"""Time the weight-gradient contractions of the C2 step (H = 512, B = 32, T = 200) and the 48000 x 2048 x 2048 layer
contraction that bench.py reports, with MN-major operands read in place and through the transposed workspace copies
(ctcb_debug_set_knob CTCB_GEMM_TC_COPY), alternated in one process.  CUDA events around REPS calls; prints one JSON line per
contraction with the plan of each path and the median over ROUNDS alternations.

    python tools/wgrad_time.py [--reps 20] [--rounds 5]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200")]

B, H, T, D, K = 32, 512, 200, 41, 62
R = T * B


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import _ctcb
    from _ctcb import lib, check, ptr
    assert torch.cuda.is_available(), "wgrad_time.py measures on the GPU"
    g = torch.Generator(device="cuda").manual_seed(1)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    feats, X1, X2, d3, d2 = rnd(R, D), rnd(R, H), rnd(R, H), rnd(R, K), rnd(R, H)
    dFor, For, dBack, Back, W2 = rnd(R, H), rnd(R, H), rnd(R, H), rnd(R, H), rnd(H, H)
    A4, B4 = rnd(48000, 2048), rnd(2048, 2048)
    st = _ctcb.current_stream()
    outs = {}

    def gemm(name, ta, tb, M, N, Kc, A, lda, Bm, ldb):
        C = outs.setdefault(name, torch.empty(M, N, device="cuda"))
        ws = outs.setdefault(name + "/ws", torch.empty(lib.ctcb_gemm_workspace_bytes(M, N, Kc), dtype=torch.uint8,
                                                       device="cuda"))
        plan = (ctypes.c_int32 * 8)()
        check(lib.ctcb_debug_gemm_plan(ta, tb, M, N, Kc, A.data_ptr(), lda, Bm.data_ptr(), ldb, 1, plan))
        run = lambda: check(lib.ctcb_gemm_f32(ta, tb, M, N, Kc, 1.0, A.data_ptr(), lda, Bm.data_ptr(), ldb, 0.0, ptr(C), N,
                                              None, 0, None, ptr(ws), ws.numel(), st))
        return run, list(plan), 2.0 * M * N * Kc

    def pair(name):
        Rm = R - B
        C = outs.setdefault(name, torch.empty(2, H, H, device="cuda"))
        ws = outs.setdefault(name + "/ws", torch.empty(lib.ctcb_gemm_pair_workspace_bytes(H, H, Rm), dtype=torch.uint8,
                                                       device="cuda"))
        A0, B0, A1, B1 = dFor[B:], For[:Rm], dBack[:Rm], Back[B:]
        plan = (ctypes.c_int32 * 8)()
        check(lib.ctcb_debug_gemm_plan(1, 0, H, H, Rm, A0.data_ptr(), H, B0.data_ptr(), H, 2, plan))
        run = lambda: check(lib.ctcb_gemm_pair_f32(1, 0, H, H, Rm, 1.0, A0.data_ptr(), A1.data_ptr(), H, B0.data_ptr(),
                                                   B1.data_ptr(), H, 0.0, ptr(C[0]), ptr(C[1]), H, ptr(ws), ws.numel(), st))
        return run, list(plan), 2 * 2.0 * H * H * Rm

    cases = {
        "dW3 = d3^T X2 (62 x 512 x 6400)": lambda: gemm("dW3", 1, 0, K, H, R, d3, K, X2, H),
        "dW2 = d2^T X1 (512 x 512 x 6400)": lambda: gemm("dW2", 1, 0, H, H, R, d2, H, X1, H),
        "d1 = d2 W2 (6400 x 512 x 512)": lambda: gemm("d1", 0, 0, R, H, H, d2, H, W2, H),
        "dWtf + dWtb (2 x 512 x 512 x 6368)": lambda: pair("rec"),
        "dW1 = d1^T feats (512 x 41 x 6400)": lambda: gemm("dW1", 1, 0, H, D, R, d2, H, feats, D),
        "layer 48000 x 2048 x 2048 (bench.py)": lambda: gemm("big", 0, 1, 48000, 2048, 2048, A4, 2048, B4, 2048),
    }
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def time_one(run, reps):
        e0.record()
        for _ in range(reps):
            run()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / reps      # us per call

    dev = torch.cuda.get_device_name(0)
    for name, make in cases.items():
        res = {"copy": [], "in_place": []}
        plans = {}
        reps = max(2, args.reps // 10) if "48000" in name else args.reps
        for rnd_ in range(args.rounds + 1):
            for mode, flag in (("copy", b"1"), ("in_place", b"0")):
                check(lib.ctcb_debug_set_knob(b"CTCB_GEMM_TC_COPY", flag))
                run, plan, flops = make()
                plans[mode] = plan
                us = time_one(run, reps)
                if rnd_ > 0:                      # round 0 warms both paths up
                    res[mode].append(us)
        check(lib.ctcb_debug_set_knob(b"CTCB_GEMM_TC_COPY", None))
        med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
        print(json.dumps({"contraction": name, "device": dev, "us_median": med, "us_all": res,
                          "speedup": med["copy"] / med["in_place"],
                          "tflops_in_place": flops / (med["in_place"] * 1e-6) / 1e12,
                          "plan {kernel,BN,stages,splits,ctas,A,B,problems}": plans}))


if __name__ == "__main__":
    main()
