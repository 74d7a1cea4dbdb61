"""GEMM rate experiment: time ctcb_gemm_f32 (operands used in place, no prep kernels) on the contractions of the C2 step
(H = 512, B = 32, T = 200) in the operand layouts the step uses, and on the 48000 x 2048 x 2048 layer contraction that
bench.py reports.  CUDA events around REPS calls, median over ROUNDS.  With --trace, one further call per shape runs with
CTCB_GEMM_TRACE=1 and the per-k-block SM clock stamps of CTA (0,0,0) are summarised (medians over its k-blocks):
    tma_wait   issue -> the producer sees the tile land
    split      tile landed -> the producer's low halves written (ready)
    mma_issue  consumers start the k-block -> its MMAs are committed
    period     consumers start one k-block -> start the next

    python tools/gemm_rate.py [--reps 20] [--rounds 5] [--trace]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200")]

B, H, T = 32, 512, 200
R = T * B


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--trace", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    import _ctcb
    from _ctcb import lib, check, ptr
    assert torch.cuda.is_available(), "gemm_rate.py measures on the GPU"
    g = torch.Generator(device="cuda").manual_seed(1)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    st = _ctcb.current_stream()

    def single(ta, tb, M, N, K):
        A = rnd(K, M) if ta else rnd(M, K)
        Bm = rnd(N, K) if tb else rnd(K, N)
        lda, ldb = (M if ta else K), (K if tb else N)
        C = torch.empty(M, N, device="cuda")
        ws = torch.empty(max(16, lib.ctcb_gemm_workspace_bytes(M, N, K)), dtype=torch.uint8, device="cuda")
        plan = (ctypes.c_int32 * 8)()
        check(lib.ctcb_debug_gemm_plan(ta, tb, M, N, K, ptr(A), lda, ptr(Bm), ldb, 1, plan))
        run = lambda: check(lib.ctcb_gemm_f32(ta, tb, M, N, K, 1.0, ptr(A), lda, ptr(Bm), ldb, 0.0, ptr(C), N, None, 0,
                                              None, ptr(ws), ws.numel(), st))
        return run, list(plan), 2.0 * M * N * K

    def pair(M, N, K):
        As, Bs = [rnd(K, M) for _ in range(2)], [rnd(K, N) for _ in range(2)]
        C = torch.empty(2, M, N, device="cuda")
        ws = torch.empty(lib.ctcb_gemm_pair_workspace_bytes(M, N, K), dtype=torch.uint8, device="cuda")
        plan = (ctypes.c_int32 * 8)()
        check(lib.ctcb_debug_gemm_plan(1, 0, M, N, K, ptr(As[0]), M, ptr(Bs[0]), N, 2, plan))
        run = lambda: check(lib.ctcb_gemm_pair_f32(1, 0, M, N, K, 1.0, ptr(As[0]), ptr(As[1]), M, ptr(Bs[0]), ptr(Bs[1]),
                                                   N, 0.0, ptr(C[0]), ptr(C[1]), N, ptr(ws), ws.numel(), st))
        return run, list(plan), 2 * 2.0 * M * N * K

    cases = {
        "C2 forward h W^T (6400 x 512 x 512, A and B K-major)": lambda: single(0, 1, R, H, H),
        "C2 delta d W (6400 x 512 x 512, B MN-major)": lambda: single(0, 0, R, H, H),
        "C2 dW = d^T h (512 x 512 x 6400, A and B MN-major)": lambda: single(1, 0, H, H, R),
        "C2 recurrent pair (2 x 512 x 512 x 6368, A and B MN-major)": lambda: pair(H, H, R - B),
        "layer 48000 x 2048 x 2048 (A and B K-major)": lambda: single(0, 1, 48000, 2048, 2048),
    }
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev = torch.cuda.get_device_name(0)
    for name, make in cases.items():
        run, plan, flops = make()
        reps = max(2, args.reps // 10) if "48000" in name else args.reps
        for _ in range(3):
            run()
        us = []
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            us.append(e0.elapsed_time(e1) * 1e3 / reps)
        med = sorted(us)[len(us) // 2]
        rec = {"contraction": name, "device": dev, "us_median": med, "us_all": us, "tflops_fp32_equivalent": flops / med / 1e6,
               "plan {kernel,BN,stages,splits,ctas,A,B,problems}": plan}
        if args.trace:
            check(lib.ctcb_debug_set_knob(b"CTCB_GEMM_TRACE", b"1"))
            run()
            torch.cuda.synchronize()
            check(lib.ctcb_debug_set_knob(b"CTCB_GEMM_TRACE", None))
            buf = (ctypes.c_ulonglong * (64 * 8))()
            if lib.ctcb_debug_gemm_trace(buf):
                s = np.array(buf, dtype=np.int64).reshape(64, 8)
                n = int(np.count_nonzero(s[:, 3]))
                s = s[:n]
                med_ = lambda x: float(np.median(x)) if len(x) else None
                rec["trace_clocks"] = {"k_blocks": n, "tma_wait": med_(s[:, 1] - s[:, 0]), "split": med_(s[:, 2] - s[:, 1]),
                                       "mma_issue": med_(s[:, 4] - s[:, 3]), "period": med_(np.diff(s[:, 3])),
                                       "consumer_waits_after_ready": med_(s[:, 3] - s[:, 2])}
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
