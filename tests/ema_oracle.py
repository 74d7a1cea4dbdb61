"""Float64 restatement of the weight average of include/ctcb200.h (ctcb_ema_update_f32), next to the adaptive rules of
tests/optim_oracle.py, whose step number it shares: t = max(1, *step)."""
import numpy as np

from optim_oracle import step_number


def ema_decay(d, t):
    """d_t = min(d, 1 - 1/t) of the float32 decay d at step t (values below 1 taken as 1), in float64 and rounded to
    float32 once, as ctcb_ema_update_f32 computes it."""
    return np.float64(np.float32(min(np.float64(np.float32(d)), 1.0 - 1.0 / step_number(t))))


def ema_update(a, w, d, t, n_valid=None):
    """The weight average after a step, in float64: w + d_t (a - w) of the float32 a and w (a when n_valid reads 0)."""
    a = np.asarray(a, dtype=np.float32).astype(np.float64)
    w = np.asarray(w, dtype=np.float32).astype(np.float64)
    if n_valid is not None and np.float32(n_valid) == 0:
        return a
    return w + ema_decay(d, t) * (a - w)


def ulps(x, y):
    """Element-wise distance in units in the last place between float32 arrays (0 for +0.0 against -0.0)."""
    def key(v):
        i = np.ascontiguousarray(v, dtype=np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(x) - key(y))
