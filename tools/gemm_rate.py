"""GEMM rate experiment: time ctcb_gemm_f32 on large NT problems (operands used in place, no prep kernels)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200")]
import numpy as np, torch
import _ctcb
from _ctcb import lib, check, ptr
for (M, N, K) in [(6400, 512, 512), (16384, 2048, 2048), (16384, 2048, 256)]:
    A = torch.randn(M, K, device="cuda"); B = torch.randn(N, K, device="cuda"); C = torch.empty(M, N, device="cuda")
    ws = torch.empty(max(16, lib.ctcb_gemm_workspace_bytes(M, N, K)), dtype=torch.uint8, device="cuda")
    st = _ctcb.current_stream()
    def run():
        check(lib.ctcb_gemm_f32(0, 1, M, N, K, 1.0, ptr(A), K, ptr(B), K, 0.0, ptr(C), N, None, 0, None, ptr(ws), ws.numel(), st))
    for _ in range(3): run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): run()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print("M=%d N=%d K=%d: %.3f ms  %.1f TFLOP/s fp32-equivalent" % (M, N, K, ms, 2.0 * M * N * K / ms / 1e9), flush=True)
