"""Float64 restatement of the adaptive update rules of include/ctcb200.h (ctcb_adagrad_step_f32, ctcb_adam_step_f32),
next to the Nesterov step of oracle/brnn_oracle.py (sgd_step).

Each function takes the kernel's own float32 inputs -- w, the state(s), the reduced gradient g, gnorm^2, the step
counter t and n_valid -- and computes the step in float64.  It returns the new values and, for the element-wise error
bound of the GPU tests, S: the sum of the magnitudes of the terms of each new value's formula, so that a float32
evaluation of that formula is within a few units of 2^-24 * S of the float64 one:
  * a state:  S = beta*|s| + (1-beta)*|g_c| (or its square); AdaGrad's r: gamma_t*r + g_c^2;
  * w:        S = |w| + the magnitude of the step with its numerator's terms taken in magnitude: |w| + |dw| for AdaGrad,
              |w| + alpha*(S_m/(1-b1^t)) / (sqrt(v_hat)+eps) for Adam -- |w| + |dw| unless m cancels, in which case
              the float32 m, and with it dw, carries an error of order 2^-24 * S_m rather than 2^-24 * |m|.

The AdaGrad rule is the reference's branch (ctc_fast/sgd.py:143-158) with cudamat's add_pow(dwt, dw, 2, alpha=gamma,
target=dwt) read as r <- gamma*r + g^2 and delta = 1e-10 under the square root only."""
import numpy as np

ADAGRAD_DELTA = 1e-10


def step_number(t):
    """The step the rules use: the counter's value, values below 1 taken as 1."""
    return max(1, int(t))


def clip_scale(gnorm2, max_gnorm):
    """c = min(1, maxGNorm / sqrt(gnorm^2)) of the float32 inputs, in float64."""
    gn = np.sqrt(np.float64(np.float32(gnorm2)))
    mx = np.float64(np.float32(max_gnorm))
    return mx / gn if gn > mx else 1.0


def adagrad_gamma(t):
    """gamma_t = 1 - 1/(0.01 t + 1): the forgetting factor of AdaGrad's squared-gradient sum, tending to 1."""
    return 1.0 - 1.0 / (0.01 * step_number(t) + 1.0)


def _f64(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def adagrad_step(w, r, g, alpha, max_gnorm, gnorm2, t, n_valid=None):
    """-> dict(w, r, S_w, S_r) in float64."""
    w, r, g = _f64(w), _f64(r), _f64(g)
    if n_valid is not None and np.float32(n_valid) == 0:
        return dict(w=w, r=r, S_w=np.abs(w), S_r=np.abs(r))
    alpha = np.float64(np.float32(alpha))
    gc = clip_scale(gnorm2, max_gnorm) * g
    gamma = adagrad_gamma(t)
    r_new = gamma * r + gc * gc
    dw = alpha * gc / np.sqrt(r_new + ADAGRAD_DELTA)
    return dict(w=w - dw, r=r_new, S_w=np.abs(w) + np.abs(dw), S_r=gamma * np.abs(r) + gc * gc)


def adam_step(w, m, v, g, alpha, beta1, beta2, eps, max_gnorm, gnorm2, t, n_valid=None):
    """-> dict(w, m, v, S_w, S_m, S_v) in float64."""
    w, m, v, g = _f64(w), _f64(m), _f64(v), _f64(g)
    if n_valid is not None and np.float32(n_valid) == 0:
        return dict(w=w, m=m, v=v, S_w=np.abs(w), S_m=np.abs(m), S_v=np.abs(v))
    alpha, b1, b2, eps = (np.float64(np.float32(x)) for x in (alpha, beta1, beta2, eps))
    tt = step_number(t)
    gc = clip_scale(gnorm2, max_gnorm) * g
    m_new = b1 * m + (1.0 - b1) * gc
    v_new = b2 * v + (1.0 - b2) * gc * gc
    bc1, bc2 = 1.0 - b1 ** tt, 1.0 - b2 ** tt
    den = np.sqrt(v_new / bc2) + eps
    dw = alpha * (m_new / bc1) / den
    S_m = b1 * np.abs(m) + (1.0 - b1) * np.abs(gc)
    return dict(w=w - dw, m=m_new, v=v_new, S_w=np.abs(w) + alpha * (S_m / bc1) / den, S_m=S_m,
                S_v=b2 * np.abs(v) + (1.0 - b2) * gc * gc)


def error_ratio(x, want, S):
    """max |x - x64| / (2^-24 * S + 2^-149): the measured constant c of the bound |x - x64| <= c * 2^-24 * S (the
    absolute 2^-149 counts only where the value is zero or subnormal)."""
    err = np.abs(np.asarray(x, dtype=np.float64) - want)
    return float(np.max(err / (2.0 ** -24 * S + 2.0 ** -149))) if err.size else 0.0
