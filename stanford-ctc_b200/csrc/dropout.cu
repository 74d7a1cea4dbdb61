// dropout.cu -- inverted dropout of a ReLU hidden layer's activations, in place, and the device step counter.
//
// The mask (defined once, at ctcb_brnn_set_dropout in include/ctcb200.h; the tests restate it in NumPy):
// unit j of frame t of minibatch utterance g in hidden layer `layer`, at optimisation step `step`, is kept iff
//     Philox4x32-10(counter = (step mod 2^32, g mod 2^32, t, (layer << 24) | (j / 4)),
//                   key = (seed mod 2^32, seed >> 32))[j % 4] >= thr
// and a kept unit becomes x * scale (one fp32 multiply), a dropped one 0.  One Philox call covers a float4 of units.
// The step is read from device memory, so a captured CUDA graph draws a new mask whenever the counter moves.
#include "common.cuh"
#include <curand_philox4x32_x.h>

namespace ctcb {

namespace {
__device__ __forceinline__ float keep(uint32_t r, uint32_t thr, float x, float scale) { return r >= thr ? x * scale : 0.f; }

// X: time-major [Tmax][B][H]; row r = t * B + u, utterance u of this call is minibatch utterance first + stride * u.
// One thread per (row, group of four units); VEC: H % 4 == 0, so every group is one aligned float4.
template <bool VEC>
__global__ void dropout_inplace_kernel(float *__restrict__ X, int64_t R, int B, int H, int layer, uint2 key,
                                       const int64_t *__restrict__ step, int64_t first, int64_t stride, uint32_t thr,
                                       float scale) {
    const int Q = (H + 3) / 4;
    const int64_t n = R * Q;
    const uint32_t s32 = (uint32_t)(*step);
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx / Q;
        const int q = (int)(idx - r * Q);
        const int64_t t = r / B;
        const int64_t u = r - t * B;
        const int64_t g = first + stride * u;
        const uint4 c = curand_Philox4x32_10(make_uint4(s32, (uint32_t)g, (uint32_t)t, ((uint32_t)layer << 24) | (uint32_t)q), key);
        float *row = X + r * H;
        if (VEC) {
            float4 v = reinterpret_cast<float4 *>(row)[q];
            v.x = keep(c.x, thr, v.x, scale);
            v.y = keep(c.y, thr, v.y, scale);
            v.z = keep(c.z, thr, v.z, scale);
            v.w = keep(c.w, thr, v.w, scale);
            reinterpret_cast<float4 *>(row)[q] = v;
        } else {
            const int j0 = 4 * q;
            const uint32_t cs[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (j0 + k < H) row[j0 + k] = keep(cs[k], thr, row[j0 + k], scale);
        }
    }
}

__global__ void advance_kernel(int64_t *step) { *step += 1; }
}  // namespace

int run_dropout(float *X, int64_t R, int B, int H, int layer, uint64_t seed, const int64_t *step, int64_t first,
                int64_t stride, uint32_t thr, float scale, cudaStream_t st) {
    const int64_t n = R * ((H + 3) / 4);
    if (n <= 0) return CTCB_OK;
    const int threads = 256;
    const int64_t want = (n + threads - 1) / threads;
    const int64_t cap = (int64_t)num_sms() * 16;        // grid-stride beyond ~16 blocks per SM
    const unsigned blocks = (unsigned)(want < cap ? want : cap);
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    if (H % 4 == 0)
        dropout_inplace_kernel<true><<<blocks, threads, 0, st>>>(X, R, B, H, layer, key, step, first, stride, thr, scale);
    else
        dropout_inplace_kernel<false><<<blocks, threads, 0, st>>>(X, R, B, H, layer, key, step, first, stride, thr, scale);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb

extern "C" int ctcb_dropout_advance(int64_t *step, void *stream) {
    if (!step) return ctcb::set_error(CTCB_EINVAL, "ctcb_dropout_advance: null step counter");
    ctcb::advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}
