"""weight_noise_oracle.py -- TEST INFRASTRUCTURE ONLY: a NumPy restatement of the Gaussian weight noise
(ctcb_brnn_set_weight_noise, include/ctcb200.h).

Element e of a noised matrix at optimisation step s, q = e // 4, j = e % 4, draws the Philox4x32-10 block (net_oracle's)
of the counter (s mod 2^32, q mod 2^32, 1, 0) under the key (seed mod 2^32, seed >> 32); (a, b) = (r0, r1) for j < 2,
(r2, r3) otherwise; u1 = (a + 1) 2^-32, u2 = b 2^-32, rho = sqrt(-2 ln u1), z = rho cos(2 pi u2) for even j and
rho sin(2 pi u2) for odd j, all in float64; w' = w + float32(sigma z).  Every element outside the noised ranges is copied
bit for bit.  cos(2 pi u2) and sin(2 pi u2) are evaluated after an exact reduction of 2 u2 to a quarter turn, so they
keep their relative accuracy near their zeros, as sincospi does."""
import numpy as np

from net_oracle import philox4x32_10

M32 = 0xFFFFFFFF


def counters(step, q):
    """(n, 4) uint64: the Philox counters of quads q at `step`."""
    q = np.asarray(q, dtype=np.uint64).reshape(-1)
    return np.stack([np.full_like(q, int(step) & M32), q & np.uint64(M32), np.ones_like(q), np.zeros_like(q)], axis=-1)


def draws(seed, step, q):
    """(n, 4) uint32: the Philox blocks of quads q at `step`."""
    return philox4x32_10(counters(step, q), (int(seed) & M32, (int(seed) >> 32) & M32))


def sincos_2pi(u2):
    """(sin 2 pi u2, cos 2 pi u2) in float64 for u2 = b 2^-32: x = 2 u2 = n / 2 + r exactly, |r| <= 1/4."""
    x = 2.0 * np.asarray(u2, dtype=np.float64)
    n = np.rint(2.0 * x)
    r = x - 0.5 * n                                   # exact: x has at most 33 significant bits
    s, c = np.sin(np.pi * r), np.cos(np.pi * r)
    k = n.astype(np.int64) % 4                        # quarter turns
    sin = np.select([k == 0, k == 1, k == 2], [s, c, -s], -c)
    cos = np.select([k == 0, k == 1, k == 2], [c, -s, -c], s)
    return sin, cos


def normals(seed, step, lo, hi):
    """float64 z of elements lo .. hi - 1 (lo a multiple of 4)."""
    e = np.arange(lo, hi, dtype=np.int64)
    q0 = lo // 4
    r = draws(seed, step, np.arange(q0, (hi + 3) // 4, dtype=np.uint64))[e // 4 - q0]
    j = e % 4
    a = np.where(j < 2, r[:, 0], r[:, 2]).astype(np.float64)
    b = np.where(j < 2, r[:, 1], r[:, 3]).astype(np.float64)
    u1 = (a + 1.0) * 2.0 ** -32
    u2 = b * 2.0 ** -32
    rho = np.sqrt(-2.0 * np.log(u1))
    sin, cos = sincos_2pi(u2)
    return np.where(j % 2 == 0, rho * cos, rho * sin)


def terms(sigma, seed, step, lo, hi):
    """float32 noise terms float32(sigma z) of elements lo .. hi - 1."""
    return (np.float64(np.float32(sigma)) * normals(seed, step, lo, hi)).astype(np.float32)


def apply(params, ranges, sigma, seed, step):
    """params (float32, flat) with the noise of `step` added inside the (lo, hi) ranges: a copy."""
    out = np.array(params, dtype=np.float32, copy=True)
    for lo, hi in ranges:
        out[lo:hi] = out[lo:hi] + terms(sigma, seed, step, lo, hi)
    return out


def cfg_ranges(cfg):
    """The (lo, hi) element ranges of the noised matrices of a ctcb_brnn_config: the even tensors below nreg, the ones
    ctcb_brnn_apply_l2_f32 regularises (W of every map, then every recurrent matrix)."""
    import ctypes
    from _ctcb import lib, check
    N, nt = cfg.numLayers, 0
    if 0 < cfg.temporalLayer <= cfg.numLayers:
        nt = max(1, cfg.numTemporal)
    nreg = 2 * (N + 1) + nt * (2 if cfg.unidirectional else 4)
    off, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    out = []
    for idx in range(0, nreg, 2):
        check(lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), idx, ctypes.byref(off), ctypes.byref(r), ctypes.byref(c)))
        out.append((off.value, off.value + r.value * c.value))
    return out
