"""TF32 mode against the fp32-faithful default, alternated in one run on one GPU:

  gemm    the tools/gemm_rate.py contractions (C2 shapes and the 48000 x 2048 x 2048 layer) through ctcb_gemm_f32 and
          ctcb_gemm_tf32: CUDA events around REPS calls, median over ROUNDS, as TFLOP/s of the product's 2 M N K and as a
          share of the H100 SXM data sheet's 495 TFLOP/s dense TF32 (a data-sheet figure, not a measured peak); with the
          CTCB_GEMM_TRACE clocks per k-block of CTA (0,0,0) (medians over its k-blocks, as gemm_rate.py --trace);
  sweep   the tensor-core ReLU sweep alone (ctcb_brnn_sweep_f32 / _tf32, forward and BPTT, both directions) at the C3
          (H 1024, B 128, T 800) and C4 (H 2048, B 32, T 1500) widths of one GPU;
  step    whole SGD.step_device steps (graph replay, as bench.py times them) of the C2, C3 and C4 nets on one GPU
          (bench.py CONFIGS; C4 at its per-GPU batch of 32), a net per mode from the same initial parameters.

The card's name, power limit and largest SM clock are read in the same run (nvidia-smi --query-gpu).  One JSON line per
measurement.

    python tools/tf32_time.py [--rounds 5] [--only gemm,sweep,step]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200")]

TF32_DENSE_TFLOPS = 495.0      # NVIDIA H100 SXM data sheet, dense TF32


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def _median(x):
    return sorted(x)[len(x) // 2]


def _alternate(runs, reps, rounds):
    """{mode: [us per call per round]}, the modes alternated within every round."""
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for run in runs.values():          # (a step is captured into a graph at its third call)
        for _ in range(4):
            run()
    out = {m: [] for m in runs}
    for _ in range(rounds):
        for m, run in runs.items():
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            out[m].append(e0.elapsed_time(e1) * 1e3 / reps)
    return out


def _trace(run):
    import numpy as np
    from _ctcb import lib, check
    check(lib.ctcb_debug_set_knob(b"CTCB_GEMM_TRACE", b"1"))
    run()
    import torch
    torch.cuda.synchronize()
    check(lib.ctcb_debug_set_knob(b"CTCB_GEMM_TRACE", None))
    buf = (ctypes.c_ulonglong * (64 * 8))()
    if not lib.ctcb_debug_gemm_trace(buf):
        return None
    s = np.array(buf, dtype=np.int64).reshape(64, 8)
    s = s[:int(np.count_nonzero(s[:, 3]))]
    med = lambda x: float(np.median(x)) if len(x) else None      # noqa: E731
    return {"k_blocks": len(s), "tma_wait": med(s[:, 1] - s[:, 0]), "split_or_round": med(s[:, 2] - s[:, 1]),
            "mma_issue": med(s[:, 4] - s[:, 3]), "period": med(np.diff(s[:, 3])),
            "consumer_waits_after_ready": med(s[:, 3] - s[:, 2])}


def gemm(args, dev):
    import torch
    import _ctcb
    from _ctcb import lib, check, ptr
    B, H, T = 32, 512, 200
    R = T * B
    g = torch.Generator(device="cuda").manual_seed(1)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)      # noqa: E731
    st = _ctcb.current_stream()

    def single(ta, tb, M, N, K):
        A = rnd(K, M) if ta else rnd(M, K)
        Bm = rnd(N, K) if tb else rnd(K, N)
        lda, ldb = (M if ta else K), (K if tb else N)
        C = torch.empty(M, N, device="cuda")
        ws = torch.empty(max(16, lib.ctcb_gemm_workspace_bytes(M, N, K)), dtype=torch.uint8, device="cuda")
        runs, plans = {}, {}
        for mode, fn, pfn in (("fp32", lib.ctcb_gemm_f32, lib.ctcb_debug_gemm_plan),
                              ("tf32", lib.ctcb_gemm_tf32, lib.ctcb_debug_gemm_plan_tf32)):
            plan = (ctypes.c_int32 * 8)()
            check(pfn(ta, tb, M, N, K, ptr(A), lda, ptr(Bm), ldb, 1, plan))
            plans[mode] = list(plan)
            runs[mode] = (lambda fn=fn: check(fn(ta, tb, M, N, K, 1.0, ptr(A), lda, ptr(Bm), ldb, 0.0, ptr(C), N, None,
                                                 0, None, ptr(ws), ws.numel(), st)))
        return runs, plans, 2.0 * M * N * K

    def pair(M, N, K):
        As, Bs = [rnd(K, M) for _ in range(2)], [rnd(K, N) for _ in range(2)]
        C = torch.empty(2, M, N, device="cuda")
        ws = torch.empty(lib.ctcb_gemm_pair_workspace_bytes(M, N, K), dtype=torch.uint8, device="cuda")
        runs, plans = {}, {}
        for mode, fn, pfn in (("fp32", lib.ctcb_gemm_pair_f32, lib.ctcb_debug_gemm_plan),
                              ("tf32", lib.ctcb_gemm_pair_tf32, lib.ctcb_debug_gemm_plan_tf32)):
            plan = (ctypes.c_int32 * 8)()
            check(pfn(1, 0, M, N, K, ptr(As[0]), M, ptr(Bs[0]), N, 2, plan))
            plans[mode] = list(plan)
            runs[mode] = (lambda fn=fn: check(fn(1, 0, M, N, K, 1.0, ptr(As[0]), ptr(As[1]), M, ptr(Bs[0]),
                                                 ptr(Bs[1]), N, 0.0, ptr(C[0]), ptr(C[1]), N, ptr(ws), ws.numel(), st)))
        return runs, plans, 2 * 2.0 * M * N * K

    cases = {
        "C2 forward h W^T (6400 x 512 x 512, A and B K-major)": lambda: single(0, 1, R, H, H),
        "C2 delta d W (6400 x 512 x 512, B MN-major)": lambda: single(0, 0, R, H, H),
        "C2 dW = d^T h (512 x 512 x 6400, A and B MN-major)": lambda: single(1, 0, H, H, R),
        "C2 recurrent pair (2 x 512 x 512 x 6368, A and B MN-major)": lambda: pair(H, H, R - B),
        "C3 dW = d^T h (1024 x 1024 x 102400, A and B MN-major)": lambda: single(1, 0, 1024, 1024, 102400),
        "layer 48000 x 2048 x 2048 (A and B K-major)": lambda: single(0, 1, 48000, 2048, 2048),
        "C4 delta d W (48000 x 2048 x 2048, B MN-major)": lambda: single(0, 0, 48000, 2048, 2048),
    }
    for name, make in cases.items():
        runs, plans, flops = make()
        reps = max(2, args.reps // 10) if "48000" in name or "102400" in name else args.reps
        us = _alternate(runs, reps, args.rounds)
        rec = {"gemm": name, "device": dev, "plan {kernel,BN,stages,splits,ctas,A,B,problems}": plans}
        for m in runs:
            med = _median(us[m])
            rec[m] = {"us_median": med, "us_all": us[m], "tflops": flops / med / 1e6,
                      "share_of_datasheet_495_dense_tf32": flops / med / 1e6 / TF32_DENSE_TFLOPS,
                      "trace_clocks": _trace(runs[m])}
        rec["tf32_speedup"] = _median(us["fp32"]) / _median(us["tf32"])
        print(json.dumps(rec), flush=True)
        del runs
        torch.cuda.empty_cache()


def sweep(args, dev):
    import numpy as np
    import torch
    import _ctcb
    from _ctcb import lib, check, ptr
    st = _ctcb.current_stream()
    for label, H, B, T in (("C3", 1024, 128, 800), ("C4", 2048, 32, 1500)):
        rng = np.random.RandomState(3)
        s = 0.9 / np.sqrt(H / 3.0)
        dv = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()      # noqa: E731
        W = [dv(rng.uniform(-s, s, (H, H))) for _ in range(2)]
        pre = dv(rng.randn(T, B, H) + 0.3)
        lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
        out = [torch.empty(T, B, H, device="cuda") for _ in range(2)]
        d = [torch.empty(T, B, H, device="cuda") for _ in range(2)]
        n = lib.ctcb_brnn_sweep_workspace_bytes(H, B)
        ws = torch.zeros(n, dtype=torch.uint8, device="cuda")
        runs, plans = {}, {}
        for mode, fn, pfn in (("fp32", lib.ctcb_brnn_sweep_f32, lib.ctcb_debug_sweep_plan),
                              ("tf32", lib.ctcb_brnn_sweep_tf32, lib.ctcb_debug_sweep_plan_tf32)):
            plan = (ctypes.c_int32 * 8)()
            check(pfn(H, B, 2, plan))
            plans[mode] = list(plan)
            for m in (0, 1):
                runs["%s_%s" % (mode, ("forward", "bptt")[m])] = (
                    lambda fn=fn, m=m: check(fn(m, T, B, H, ptr(lens), ptr(pre), ptr(W[0]), ptr(W[1]),
                                                ptr(d[0] if m else out[0]), ptr(d[1] if m else out[1]),
                                                ptr(out[0]) if m else None, ptr(out[1]) if m else None, 20.0,
                                                ptr(ws), n, st)))
        runs["fp32_forward"]()           # the BPTT reads forward states
        us = _alternate(runs, 3, args.rounds)
        rec = {"sweep": "%s: H %d, B %d, T %d, two directions" % (label, H, B, T), "device": dev,
               "plan {kernel,KI,CS,NS,NP,stages,partial_own,-}": plans}
        for m in runs:
            rec[m] = {"ms_median": _median(us[m]) / 1e3, "us_per_step": _median(us[m]) / T}
        for ph in ("forward", "bptt"):
            rec["tf32_speedup_" + ph] = _median(us["fp32_" + ph]) / _median(us["tf32_" + ph])
        print(json.dumps(rec), flush=True)
        del runs, W, pre, out, d, ws
        torch.cuda.empty_cache()


def step(args, dev):
    import numpy as np
    import torch
    import bench
    import nnets.brnnet as rnnet
    import sgd
    for key, Bl in (("c2", 32), ("c3", 128), ("c4", 32)):
        c = bench.CONFIGS[key]
        datas, labels = bench.make_batch(c, Bl, seed=33)
        nets = {}
        for mode in ("fp32", "tf32"):
            np.random.seed(33)
            nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=Bl,
                            maxLabels=c["L"], tf32=(mode == "tf32"))
            nn.initParams()
            opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=Bl, verbose=False)
            opt.it = 11                                  # past the momentum warm-up: one graph
            nets[mode] = (nn, opt, nn._batch.pack(datas, labels).upload())
        stream = torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            def make(mode):
                nn, opt, batch = nets[mode]

                def run():
                    opt.it += 1
                    opt.step_device(batch, opt._momentum_now())
                return run
            runs = {m: make(m) for m in nets}
            reps = 2 if key == "c4" else 5
            us = _alternate(runs, reps, args.rounds)
        rec = {"step": c["name"] + " (one GPU, per-GPU batch %d)" % Bl, "device": dev}
        for m in runs:
            rec[m] = {"ms_median": _median(us[m]) / 1e3, "ms_all": [u / 1e3 for u in us[m]]}
        rec["tf32_speedup"] = _median(us["fp32"]) / _median(us["tf32"])
        print(json.dumps(rec), flush=True)
        del nets, runs
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", default="gemm,sweep,step")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "tf32_time.py measures on the GPU"
    dev = card()
    print(json.dumps({"card": dev}), flush=True)
    for part in args.only.split(","):
        {"gemm": gemm, "sweep": sweep, "step": step}[part](args, dev)


if __name__ == "__main__":
    main()
