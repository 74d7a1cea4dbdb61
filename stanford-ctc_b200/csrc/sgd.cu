// sgd.cu -- optimiser arithmetic on the flat parameter vector.
//
// Replaces, per step, the ~16(N+3) cudamat launches and 2(N+3) blocking euclid_norm() reads of
//   ctc_fast/sgd.py:91-100   (Nesterov look-ahead / undo via NNet.updateParams)
//   ctc_fast/sgd.py:103-107  (global gradient norm)
//   ctc_fast/sgd.py:130-140  (clip scale, velocity update)
//   ctc_fast/sgd.py:161 and nnets/brnnet.py:251-256 (w += v)
// with one axpy, one two-stage sum of squares and one fused update kernel; the clip scale is
// computed on the device from the reduced norm, so the step never synchronises with the host.
// AdaGrad (ctc_fast/sgd.py:143-158) and Adam, not in the reference's working code, are one fused kernel each; the
// exponential moving average of the weights is one more pass behind whichever rule ran.
#include <cmath>
#include "common.cuh"

namespace ctcb {

__global__ void axpy_kernel(float *__restrict__ w, const float *__restrict__ u, float scale, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        w[i] = fmaf(scale, u[i], w[i]);   // add_mult: w += scale*u
}

constexpr int SS_BLOCKS = 512;

__global__ void sumsq_stage1(const float *__restrict__ g, int64_t n, double *__restrict__ partial) {
    double s = 0.0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float v = g[i];
        s += (double)v * (double)v;
    }
    __shared__ double sh[256];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}

// out = (accumulate ? out : 0) + scale * sum(partials)
__global__ void sumsq_stage2(const double *__restrict__ partial, int nparts, float *out, float scale, int accumulate) {
    __shared__ double sh[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < nparts; i += blockDim.x) s += partial[i];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = (accumulate ? out[0] : 0.f) + scale * (float)sh[0];
}

__global__ void nesterov_kernel(float *__restrict__ w, float *__restrict__ v, const float *__restrict__ g, int64_t n,
                                float mom, float alpha, float max_gnorm, const float *__restrict__ gnorm2,
                                const float *__restrict__ n_valid) {
    // sgd.py:130-132: alph = alpha * maxGNorm/gnorm if gnorm > maxGNorm
    const float gn = sqrtf(gnorm2[0]);
    const float alph = (gn > max_gnorm) ? alpha * (max_gnorm / gn) : alpha;
    const bool all_skipped = (n_valid != nullptr) && (n_valid[0] == 0.f);   // sgd.py:109-111
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float wi = w[i], vi = v[i];
        wi = fmaf(-mom, vi, wi);          // sgd.py:100  undo the look-ahead
        if (all_skipped) { w[i] = wi; continue; }
        vi = vi * mom;                    // sgd.py:136  vw.mult(mom)
        vi = fmaf(-alph, g[i], vi);       // sgd.py:138  vw.add_mult(dw, -alph)
        wi = wi + vi;                     // sgd.py:161  updateParams(1.0, velocity)
        w[i] = wi;
        v[i] = vi;
    }
}

// The adaptive rules (include/ctcb200.h: ctcb_adagrad_step_f32, ctcb_adam_step_f32).  Both clip the gradient itself,
// g_c = c*g with c = min(1, maxGNorm/sqrt(*gnorm2)), read the step number t = max(1, *step) from device memory (a CUDA
// graph replay sees the counter's current value) and do no look-ahead.  Per-step scalars are computed in float64 once
// per thread and rounded to float32; the element arithmetic is float32.
__device__ __forceinline__ float clip_scale(const float *gnorm2, float max_gnorm) {
    const float gn = sqrtf(gnorm2[0]);
    return (gn > max_gnorm) ? max_gnorm / gn : 1.f;
}

__device__ __forceinline__ double step_number(const int64_t *step) {
    const int64_t t = step[0];
    return (double)(t < 1 ? 1 : t);
}

// r <- gamma_t*r + g_c^2,  gamma_t = 1 - 1/(0.01 t + 1);  w <- w - alpha*g_c/sqrt(r + 1e-10)      20 B per parameter
__global__ void adagrad_kernel(float *__restrict__ w, float *__restrict__ r, const float *__restrict__ g, int64_t n,
                               float alpha, float max_gnorm, const float *__restrict__ gnorm2,
                               const float *__restrict__ n_valid, const int64_t *__restrict__ step) {
    if (n_valid != nullptr && n_valid[0] == 0.f) return;                    // sgd.py:109-111
    const float c = clip_scale(gnorm2, max_gnorm);
    const float gamma = (float)(1.0 - 1.0 / (0.01 * step_number(step) + 1.0));
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float gc = c * g[i];
        const float ri = fmaf(gamma, r[i], gc * gc);
        r[i] = ri;
        w[i] = fmaf(-alpha, gc / sqrtf(ri + 1e-10f), w[i]);
    }
}

// m <- b1*m + (1-b1)*g_c;  v <- b2*v + (1-b2)*g_c^2;  w <- w - alpha*(m/(1-b1^t)) / (sqrt(v/(1-b2^t)) + eps)
// (Kingma & Ba, Algorithm 1)                                                                            28 B per parameter
__global__ void adam_kernel(float *__restrict__ w, float *__restrict__ m, float *__restrict__ v,
                            const float *__restrict__ g, int64_t n, float alpha, float beta1, float beta2, float eps,
                            float max_gnorm, const float *__restrict__ gnorm2, const float *__restrict__ n_valid,
                            const int64_t *__restrict__ step) {
    if (n_valid != nullptr && n_valid[0] == 0.f) return;
    const float c = clip_scale(gnorm2, max_gnorm);
    const double t = step_number(step);
    const float bc1 = (float)(1.0 - pow((double)beta1, t));
    const float bc2 = (float)(1.0 - pow((double)beta2, t));
    const float ob1 = (float)(1.0 - (double)beta1), ob2 = (float)(1.0 - (double)beta2);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float gc = c * g[i];
        const float mi = fmaf(beta1, m[i], ob1 * gc);
        const float vi = fmaf(beta2, v[i], ob2 * (gc * gc));
        m[i] = mi;
        v[i] = vi;
        w[i] = fmaf(-alpha, (mi / bc1) / (sqrtf(vi / bc2) + eps), w[i]);
    }
}

// The weight average (include/ctcb200.h: ctcb_ema_update_f32), launched after the rule's kernel on the w it wrote:
// a <- fmaf(d_t, a - w, w),  d_t = min(d, 1 - 1/t)                                                  12 B per parameter
// d_t = 0 (t <= 1) is a plain copy, so a becomes w bit for bit whatever a held (-0.0, infinities and NaN included).
__global__ void ema_kernel(float *__restrict__ a, const float *__restrict__ w, int64_t n, float decay,
                           const float *__restrict__ n_valid, const int64_t *__restrict__ step) {
    if (n_valid != nullptr && n_valid[0] == 0.f) return;
    const float d = (float)fmin((double)decay, 1.0 - 1.0 / step_number(step));
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (d == 0.f) {
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) a[i] = w[i];
        return;
    }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float wi = w[i];
        a[i] = fmaf(d, a[i] - wi, wi);
    }
}

static int ew_blocks(int64_t n) {
    int64_t b = (n + 1023) / 1024;
    const int cap = 8 * num_sms();
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

int run_sumsq(const float *g, int64_t n, float *out, float scale, int accumulate, void *scratch, cudaStream_t st) {
    int blocks = (int)((n + 255) / 256);
    if (blocks > SS_BLOCKS) blocks = SS_BLOCKS;
    if (blocks < 1) blocks = 1;
    sumsq_stage1<<<blocks, 256, 0, st>>>(g, n, (double *)scratch);
    CTCB_LAUNCH_CHECK();
    sumsq_stage2<<<1, 256, 0, st>>>((const double *)scratch, blocks, out, scale, accumulate);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb

using namespace ctcb;

extern "C" int ctcb_axpy_f32(float *w, const float *u, float scale, int64_t n, void *stream) {
    if (n <= 0) return CTCB_OK;
    if (!w || !u) return set_error(CTCB_EINVAL, "ctcb_axpy_f32: null pointer");
    ProfScope ps("sgd", (cudaStream_t)stream);
    axpy_kernel<<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>(w, u, scale, n);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

extern "C" int ctcb_sumsq_f32(const float *g, int64_t n, float *gnorm2_out, void *scratch, void *stream) {
    if (!g || !gnorm2_out || !scratch) return set_error(CTCB_EINVAL, "ctcb_sumsq_f32: null pointer");
    ProfScope ps("sgd", (cudaStream_t)stream);
    return run_sumsq(g, n, gnorm2_out, 1.0f, 0, scratch, (cudaStream_t)stream);
}

extern "C" int ctcb_sgd_nesterov_step_f32(float *w, float *v, const float *g, int64_t n, float mom, float alpha,
                                          float max_gnorm, const float *gnorm2, const float *n_valid, void *stream) {
    if (n <= 0) return CTCB_OK;
    if (!w || !v || !g || !gnorm2) return set_error(CTCB_EINVAL, "ctcb_sgd_nesterov_step_f32: null pointer");
    ProfScope ps("sgd", (cudaStream_t)stream);
    nesterov_kernel<<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>(w, v, g, n, mom, alpha, max_gnorm, gnorm2, n_valid);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

static bool valid_step_size(float alpha) { return std::isfinite(alpha) && alpha >= 0.f; }
static bool valid_beta(float beta) { return beta >= 0.f && beta < 1.f; }      // false for NaN

extern "C" int ctcb_adagrad_step_f32(float *w, float *r, const float *g, int64_t n, float alpha, float max_gnorm,
                                     const float *gnorm2, const float *n_valid, const int64_t *step, void *stream) {
    if (n <= 0) return CTCB_OK;
    if (!w || !r || !g || !gnorm2 || !step) return set_error(CTCB_EINVAL, "ctcb_adagrad_step_f32: null pointer");
    if (!valid_step_size(alpha))
        return set_error(CTCB_EINVAL, "ctcb_adagrad_step_f32: alpha=%g must be finite and >= 0", (double)alpha);
    ProfScope ps("sgd", (cudaStream_t)stream);
    adagrad_kernel<<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>(w, r, g, n, alpha, max_gnorm, gnorm2, n_valid, step);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

extern "C" int ctcb_adam_step_f32(float *w, float *m, float *v, const float *g, int64_t n, float alpha, float beta1,
                                  float beta2, float eps, float max_gnorm, const float *gnorm2, const float *n_valid,
                                  const int64_t *step, void *stream) {
    if (n <= 0) return CTCB_OK;
    if (!w || !m || !v || !g || !gnorm2 || !step) return set_error(CTCB_EINVAL, "ctcb_adam_step_f32: null pointer");
    if (!valid_step_size(alpha))
        return set_error(CTCB_EINVAL, "ctcb_adam_step_f32: alpha=%g must be finite and >= 0", (double)alpha);
    if (!valid_beta(beta1) || !valid_beta(beta2))
        return set_error(CTCB_EINVAL, "ctcb_adam_step_f32: beta1=%g, beta2=%g must be in [0, 1)", (double)beta1,
                         (double)beta2);
    if (!(eps > 0.f) || !std::isfinite(eps))
        return set_error(CTCB_EINVAL, "ctcb_adam_step_f32: eps=%g must be finite and > 0", (double)eps);
    ProfScope ps("sgd", (cudaStream_t)stream);
    adam_kernel<<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>(w, m, v, g, n, alpha, beta1, beta2, eps, max_gnorm,
                                                                gnorm2, n_valid, step);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

extern "C" int ctcb_ema_update_f32(float *avg, const float *w, int64_t n, float decay, const float *n_valid,
                                   const int64_t *step, void *stream) {
    if (n <= 0) return CTCB_OK;
    if (!avg || !w || !step) return set_error(CTCB_EINVAL, "ctcb_ema_update_f32: null pointer");
    if (!valid_beta(decay))
        return set_error(CTCB_EINVAL, "ctcb_ema_update_f32: decay=%g must be in [0, 1)", (double)decay);
    ProfScope ps("sgd", (cudaStream_t)stream);
    ema_kernel<<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>(avg, w, n, decay, n_valid, step);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}
