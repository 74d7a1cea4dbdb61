// sgd.cu -- optimiser arithmetic on the flat parameter vector.
//
// Replaces, per step, the ~16(N+3) cudamat launches and 2(N+3) blocking euclid_norm() reads of
//   ctc_fast/sgd.py:91-100   (Nesterov look-ahead / undo via NNet.updateParams)
//   ctc_fast/sgd.py:103-107  (global gradient norm)
//   ctc_fast/sgd.py:130-140  (clip scale, velocity update)
//   ctc_fast/sgd.py:161 and nnets/brnnet.py:251-256 (w += v)
// with one axpy, one two-stage sum of squares and one fused update kernel; the clip scale is
// computed on the device from the reduced norm, so the step never synchronises with the host.
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
