"""Check + time ctcb_gemm_f32 (wgmma 3xTF32 path unless CTCB_GEMM=simt) against float64 NumPy."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200")]
import numpy as np, torch
import _ctcb
from _ctcb import lib, check, ptr
rng = np.random.RandomState(0)
shapes = [(6400, 512, 512, 0, 1), (6400, 62, 512, 0, 1), (6400, 512, 62, 0, 0), (6400, 512, 512, 0, 0),
          (512, 512, 6400, 1, 0), (62, 512, 6400, 1, 0), (512, 41, 6400, 1, 0), (512, 512, 6368, 1, 0),
          (200, 130, 100, 0, 1), (128, 128, 32, 0, 1), (300, 70, 36, 1, 1)]
if len(sys.argv) > 1 and sys.argv[1] == "big":      # the C3 / C4 layer contractions (forward, delta, weight gradient)
    shapes = [(25600, 1024, 1024, 0, 1), (25600, 1024, 1024, 0, 0), (1024, 1024, 25600, 1, 0),
              (48000, 2048, 2048, 0, 1), (48000, 2048, 2048, 0, 0), (2048, 2048, 48000, 1, 0), (2048, 2048, 192000, 1, 0)]
if len(sys.argv) > 1 and sys.argv[1] == "small":    # the C2 step's contractions that stay on the exact FFMA kernel
    shapes = [(6400, 512, 41, 0, 1), (6400, 512, 62, 0, 0), (62, 512, 6400, 1, 0), (512, 41, 6400, 1, 0)]
if len(sys.argv) > 1 and sys.argv[1] == "quick":
    shapes = shapes[-3:] + shapes[:1]
for (M, N, K, ta, tb) in shapes:
    A = rng.randn(*((K, M) if ta else (M, K))).astype(np.float32)
    B = rng.randn(*((N, K) if tb else (K, N))).astype(np.float32)
    bias = rng.randn(N).astype(np.float32)
    ref = (A.T if ta else A).astype(np.float64) @ (B.T if tb else B).astype(np.float64) + bias
    dA, dB, dbias = (torch.from_numpy(x).cuda() for x in (A, B, bias))
    C = torch.zeros(M, N, device="cuda")
    nb = lib.ctcb_gemm_workspace_bytes(M, N, K)
    ws = torch.empty(max(nb, 16), dtype=torch.uint8, device="cuda")
    st = _ctcb.current_stream()
    def run():
        check(lib.ctcb_gemm_f32(ta, tb, M, N, K, 1.0, ptr(dA), A.shape[1], ptr(dB), B.shape[1], 0.0, ptr(C), N,
                                ptr(dbias), 0, None, ptr(ws), ws.numel(), st))
    run(); torch.cuda.synchronize()
    out = C.cpu().numpy().astype(np.float64)
    err = np.linalg.norm(out - ref) / np.linalg.norm(ref)
    mx = np.abs(out - ref).max()
    for _ in range(2): run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): run()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print("M=%5d N=%4d K=%5d tA=%d tB=%d  rel=%.2e maxabs=%.2e  %.3f ms  %.1f TFLOP/s(fp32-equiv)  [%s]" % (
        M, N, K, ta, tb, err, mx, ms, 2.0 * M * N * K / ms / 1e9, os.environ.get("CTCB_GEMM", "tc")), flush=True)
    if os.environ.get("CTCB_GEMM_TRACE"):
        import ctypes
        buf = (ctypes.c_uint64 * 512)()
        if lib.ctcb_debug_gemm_trace(buf):
            tr = np.frombuffer(buf, dtype=np.uint64).reshape(64, 8).astype(np.int64)
            t0 = tr[0, 0]
            print("   k-block:  TMA issued   landed  lo written  MMA saw   MMAs issued   (SM cycles from the first TMA issue)")
            for i in list(range(0, 8)) + [16, 17, 18, 19]:
                print("   %6d  %11d %8d %11d %8d %13d" % ((i,) + tuple(int(tr[i, j] - t0) for j in range(5))))
