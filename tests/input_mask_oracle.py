"""input_mask_oracle.py -- TEST INFRASTRUCTURE ONLY: a NumPy restatement of the SpecAugment masks of the input features
(ctcb_brnn_set_input_masks, include/ctcb200.h).

Utterance g at optimisation step s draws, for mask k = 0 .. mF + mT - 1, one Philox4x32-10 block (net_oracle's) of the
counter (s mod 2^32, g mod 2^32, 0, k) under the key (seed mod 2^32, seed >> 32).  The first mF masks are bands of
the nu filter-bank bins, the others spans of raw frames, both as [start, end) in Python integers (exact 64-bit
products).  A row t' < T_u of the time-major features holds c = D / nu frame slots, slot j the raw frame
clamp(t' + j - h, 0, T_u - 1), h = (c - 1) / 2; an element is +0.0 where its bin or its raw frame is masked, and every
other element, the padding rows included, is copied bit for bit."""
import numpy as np

from net_oracle import philox4x32_10

M32 = 0xFFFFFFFF


def draws(seed, step, g, n):
    """(n, 4) uint32: the Philox blocks of masks 0..n-1 of minibatch utterance g at `step`."""
    k = np.arange(n, dtype=np.uint64)
    ctr = np.stack([np.full_like(k, int(step) & M32), np.full_like(k, int(g) & M32), np.zeros_like(k), k], axis=-1)
    return philox4x32_10(ctr, (int(seed) & M32, (int(seed) >> 32) & M32))


def time_limit(Tu, Tw, p):
    """W = min(T, floor(p T_u)), the product in float64."""
    return min(int(Tw), int(np.floor(np.float64(p) * np.float64(Tu))))


def bands(seed, step, g, nu, Tu, mF, F, mT, Tw, p):
    """([(f0, f1)] of the mF frequency masks, [(t0, t1)] of the mT time masks) of utterance g with T_u frames."""
    r = draws(seed, step, g, mF + mT)
    W = time_limit(Tu, Tw, p)
    freq, time = [], []
    for k in range(mF + mT):
        r0, r1 = int(r[k, 0]), int(r[k, 1])
        if k < mF:
            w = (r0 * (F + 1)) >> 32
            a = (r1 * (nu - w + 1)) >> 32
            freq.append((a, a + w))
        else:
            w = (r0 * (W + 1)) >> 32
            a = (r1 * (Tu - w + 1)) >> 32
            time.append((a, a + w))
    return freq, time


def raw_frames(Tu, rows, c):
    """int [rows][c]: the raw frame each slot of rows 0..rows-1 holds (meaningful for rows < T_u)."""
    h = (c - 1) // 2
    t = np.arange(rows)[:, None] + np.arange(c)[None, :] - h
    return np.clip(t, 0, max(Tu - 1, 0))


def utterance_mask(Tu, rows, nu, c, freq, time):
    """bool [rows][c nu]: True where an element of the utterance's rows is zeroed."""
    fm = np.zeros(nu, dtype=bool)
    for a, b in freq:
        fm[a:b] = True
    tm = np.zeros(max(Tu, 1), dtype=bool)
    for a, b in time:
        tm[a:b] = True
    m = tm[raw_frames(Tu, rows, c)][:, :, None] | fm[None, None, :]
    m[Tu:] = False
    return m.reshape(rows, c * nu)


def batch_mask(lens, Tmax, D, nu, mF, F, mT, Tw, p, seed, step, first=0, stride=1):
    """bool [Tmax][B][D]: the masked elements of a call whose utterance u is minibatch utterance first + stride u."""
    c = D // nu
    out = np.zeros((Tmax, len(lens), D), dtype=bool)
    for u, Tu in enumerate(lens):
        freq, time = bands(seed, step, first + stride * u, nu, Tu, mF, F, mT, Tw, p)
        out[:, u, :] = utterance_mask(Tu, Tmax, nu, c, freq, time)
    return out


def apply(feats, mask):
    """feats [Tmax][B][D] float32 with the masked elements +0.0 (a copy)."""
    return np.where(mask, np.float32(0.0), feats).astype(np.float32)
