"""BASELINE.json configs[4]: CTC-kernel isolation sweep T x |l| x K -> algorithmic GB/s vs the HBM roofline.
Batch sizes are chosen so that the activations exceed L2 (50 MB on H100) where the alpha spill workspace allows.

Usage:  python tools/ctc_sweep.py [OUT.json]      (default: ctc_sweep.json in the current directory)"""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200")]
import numpy as np, torch
import ctc_fast
from _ctcb import lib
peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"hbm_gbs": 3350.0}   # H100 SXM data sheet
rows = []
for T in (100, 500, 2000, 5000):
    for L in (10, 100, 300):
        for K in (32, 62, 128):
            if T < L:
                rows.append(dict(T=T, L=L, K=K, note="infeasible (T < |l|): reference skips, sgd.py:84-88"))
                continue
            alg_per = 8.0 * K * T + 4.0 * L + 4.0
            B = int(min(65536, max(64, 6e8 / alg_per)))
            ws_per = lib.ctcb_ctc_workspace_bytes(1, T, L)
            B = int(max(16, min(B, 12e9 / ws_per)))
            g = torch.Generator(device="cuda").manual_seed(T + L + K)
            acts = torch.randn(B, T, K, device="cuda", generator=g)
            rng = np.random.RandomState(1)
            seqs = torch.from_numpy((1 + rng.randint(0, K - 1, size=(B * L))).astype(np.int32)).cuda()
            offs = torch.arange(0, (B + 1) * L, L, dtype=torch.int32, device="cuda")
            lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
            grad = torch.empty_like(acts)
            ws = torch.empty(lib.ctcb_ctc_workspace_bytes(B, T, L), dtype=torch.uint8, device="cuda")
            for _ in range(2):
                ctc_fast.ctc_loss_batch(acts, lens, seqs, offs, L, grad=grad, workspace=ws)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 3
            e0.record()
            for _ in range(reps):
                nll, _, skip = ctc_fast.ctc_loss_batch(acts, lens, seqs, offs, L, grad=grad, workspace=ws)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            gbs = B * alg_per / ms / 1e6
            rows.append(dict(T=T, L=L, K=K, B=B, ms=round(ms, 3), utt_per_s=round(B / ms * 1e3), alg_GBs=round(gbs, 1),
                             frac_hbm=round(gbs / peaks["hbm_gbs"], 4), act_MB=round(B * alg_per / 2e6, 1), skips=int(skip.sum()),
                             shape="two warps per utterance" if B <= min(8, (200 * 1024) // (384 * ((K + 29) // 32 * 32 + 2))) * torch.cuda.get_device_properties(0).multi_processor_count else "one warp per utterance"))
            print(rows[-1], flush=True)
            del acts, grad, ws
            torch.cuda.empty_cache()
json.dump(dict(peak_hbm_gbs=peaks["hbm_gbs"], rows=rows), open(sys.argv[1] if len(sys.argv) > 1 else "ctc_sweep.json", "w"), indent=1)
