"""GPU unit test of the persistent recurrent sweep on its own (ctcb_brnn_sweep_f32) against a NumPy
float64 restatement of brnnet.py:144-152 (forward) and :208-224 (BPTT), over layer sizes that take the
register-resident path (H = 128/256/512), the tensor-core path (H >= 1024) and the generic path, full and partial
utterance tiles, ragged lengths and the 20.0 clip."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _ref_forward(pre, Wf, Wb, lens, maxAct):
    T, B, H = pre.shape
    F = np.zeros_like(pre); Bk = np.zeros_like(pre)
    for b in range(B):
        Tb = lens[b]
        for t in range(Tb):
            h = pre[t, b] + (Wf @ F[t - 1, b] if t > 0 else 0.0)
            F[t, b] = np.clip(h, 0.0, maxAct)
        for t in range(Tb - 1, -1, -1):
            h = pre[t, b] + (Wb @ Bk[t + 1, b] if t + 1 < Tb else 0.0)
            Bk[t, b] = np.clip(h, 0.0, maxAct)
    return F, Bk


def _ref_bptt(d, Wf, Wb, F, Bk, lens, maxAct):
    T, B, H = d.shape
    dF = np.zeros_like(d); dB = np.zeros_like(d)
    mF = (F > 0) & (F < maxAct); mB = (Bk > 0) & (Bk < maxAct)
    for b in range(B):
        Tb = lens[b]
        for t in range(Tb - 1, -1, -1):
            dF[t, b] = mF[t, b] * (d[t, b] + (Wf.T @ dF[t + 1, b] if t + 1 < Tb else 0.0))
        for t in range(Tb):
            dB[t, b] = mB[t, b] * (d[t, b] + (Wb.T @ dB[t - 1, b] if t > 0 else 0.0))
    return dF, dB


@pytest.mark.parametrize("H,B,T", [(128, 8, 40), (128, 3, 33), (256, 9, 25), (512, 4, 30), (512, 32, 50),
                                     (1024, 16, 12), (96, 5, 20), (30, 2, 10), (64, 17, 21), (512, 16, 20),
                                     (256, 64, 10),
                                     # the tensor-core kernel (sweep_tc.cu, H >= 1024): one and two utterance splits, partial
                                     # 16-utterance tiles, the C3 / C4 per-GPU batch widths, H not a power of two
                                     (1024, 128, 10), (1024, 40, 9), (1024, 3, 7), (2048, 32, 8), (2048, 256, 5),
                                     (1536, 20, 6), (1024, 200, 5), (2048, 100, 4)])
def test_sweep_forward_and_bptt(H, B, T, cuda):
    import _ctcb
    from _ctcb import lib, check, ptr
    torch = cuda
    if H >= 1024:     # these sizes must run on the tensor-core kernel, not on the generic one
        assert lib.ctcb_sweep_uses_tensor_cores(H, B) == 1, (H, B)
    rng = np.random.RandomState(H + B)
    s = 0.9 / np.sqrt(H / 3.0)                        # spectral radius ~0.9: well conditioned
    Wf = rng.uniform(-s, s, (H, H)); Wb = rng.uniform(-s, s, (H, H))
    pre = rng.randn(T, B, H) * 2.0 + 0.5
    pre[T // 2] += 25.0                               # drive some units into the clip
    lens = rng.randint(max(1, T // 2), T + 1, size=B); lens[0] = T
    for b in range(B):
        pre[lens[b]:, b] = 0.0
    maxAct = 20.0
    F, Bk = _ref_forward(pre, Wf, Wb, lens, maxAct)
    assert (F >= maxAct).any()
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    d_pre, d_Wf, d_Wb = dev(pre), dev(Wf), dev(Wb)
    d_len = torch.from_numpy(lens.astype(np.int32)).cuda()
    oF = torch.empty(T, B, H, device="cuda"); oB = torch.empty(T, B, H, device="cuda")
    nscr = int(lib.ctcb_brnn_sweep_workspace_bytes(H, B))
    scratch = torch.zeros(nscr // 4, dtype=torch.int32, device="cuda")
    check(lib.ctcb_brnn_sweep_f32(0, T, B, H, ptr(d_len), ptr(d_pre), ptr(d_Wf), ptr(d_Wb), ptr(oF), ptr(oB), None,
                                  None, maxAct, ptr(scratch), nscr, _ctcb.current_stream()))
    torch.cuda.synchronize()
    assert scratch[:3].tolist() == [0, 0, 0], "error flag %s" % scratch[:3].tolist()
    gF, gB = oF.cpu().numpy().astype(np.float64), oB.cpu().numpy().astype(np.float64)
    assert np.isfinite(gF).all() and np.isfinite(gB).all()
    assert np.abs(gF - F).max() < 2e-4 * max(1.0, np.abs(F).max()), np.argwhere(np.abs(gF - F) > 1e-3)[:5]
    assert np.abs(gB - Bk).max() < 2e-4 * max(1.0, np.abs(Bk).max()), np.argwhere(np.abs(gB - Bk) > 1e-3)[:5]
    # BPTT on the float32 states the kernel itself produced (so the masks agree exactly)
    d = rng.randn(T, B, H)
    for b in range(B):
        d[lens[b]:, b] = 0.0
    F32, B32 = oF.cpu().numpy().astype(np.float64), oB.cpu().numpy().astype(np.float64)
    dF, dB = _ref_bptt(d, Wf, Wb, F32, B32, lens, maxAct)
    odF = torch.empty(T, B, H, device="cuda"); odB = torch.empty(T, B, H, device="cuda")
    check(lib.ctcb_brnn_sweep_f32(1, T, B, H, ptr(d_len), ptr(dev(d)), ptr(d_Wf), ptr(d_Wb), ptr(odF), ptr(odB),
                                  ptr(oF), ptr(oB), maxAct, ptr(scratch), nscr, _ctcb.current_stream()))
    torch.cuda.synchronize()
    assert scratch[:3].tolist() == [0, 0, 0], "error flag %s" % scratch[:3].tolist()
    gdF, gdB = odF.cpu().numpy().astype(np.float64), odB.cpu().numpy().astype(np.float64)
    assert np.isfinite(gdF).all() and np.isfinite(gdB).all()
    assert np.abs(gdF - dF).max() < 2e-4 * max(1.0, np.abs(dF).max()), np.argwhere(np.abs(gdF - dF) > 1e-3)[:5]
    assert np.abs(gdB - dB).max() < 2e-4 * max(1.0, np.abs(dB).max()), np.argwhere(np.abs(gdB - dB) > 1e-3)[:5]


def test_general_barrier_kernel_when_forced(cuda):
    """CTCB_SWEEP=barrier forces the L2/counter-barrier kernel for sizes the cluster kernel would take."""
    import os
    import subprocess
    import sys
    code = ("import os,sys; sys.path[:0]=[%r,%r,%r]; import pytest; "
            "sys.exit(pytest.main(['-q','-p','no:cacheprovider','-k','test_sweep_forward_and_bptt and (512-32-50 or 128-3-33 or 256-9-25)', %r]))"
            % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
               os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stanford-ctc_b200"),
               os.path.dirname(os.path.abspath(__file__)), os.path.abspath(__file__)))
    env = dict(os.environ, CTCB_SWEEP="barrier")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-500:]
