// weight_noise.cu -- Gaussian weight noise: one pass that copies the flat parameter vector and adds sigma * z to every
// element of the noised matrices.
//
// The rule is defined once, at ctcb_brnn_set_weight_noise in include/ctcb200.h (the tests restate it in NumPy): element
// e of a noised matrix at optimisation step s draws (r0, r1, r2, r3) = Philox4x32-10(counter = (s mod 2^32,
// (e / 4) mod 2^32, 1, 0), key = (seed mod 2^32, seed >> 32)); elements 4q, 4q + 1 take the Box-Muller pair of
// (r0, r1), elements 4q + 2, 4q + 3 that of (r2, r3), in float64.  Every other element is copied bit for bit.
//
// One thread per quad of four elements, grid-stride.  Every tensor starts on a quad, so a quad lies in at most one
// noised range; the ranges ascend, and each thread keeps a cursor into them that only moves forward.
#include "common.cuh"
#include <curand_philox4x32_x.h>

namespace ctcb {

// The most noised matrices of a net: the even tensors below nreg (NetTable), 2 * 65 + 4 * 64 of them at most.
constexpr int WN_MAX_RANGES = 193;

namespace {
constexpr int WN_THREADS = 256;

// [lo, hi) element ranges of the noised matrices, ascending; lo is a multiple of 4.  Passed by value: 3 KB of kernel
// parameters, read through the constant bank.
struct NoiseRanges {
    int64_t lo[WN_MAX_RANGES], hi[WN_MAX_RANGES];
    int n;
};
static_assert(sizeof(NoiseRanges) + 64 <= 4096, "the ranges must fit the classic 4 KB of kernel parameters");

// float32(sigma * z) for z = rho cos(2 pi u2) (odd = false) or rho sin(2 pi u2) (odd = true) of the pair (a, b)
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, double sigma, float &even, float &odd) {
    const double u1 = ((double)a + 1.0) * 0x1p-32;      // (0, 1]: the logarithm is finite
    const double u2 = (double)b * 0x1p-32;
    const double rho = sqrt(-2.0 * log(u1));
    double s, c;
    sincospi(2.0 * u2, &s, &c);
    const double z0 = rho * c, z1 = rho * s;
    even = (float)(sigma * z0);
    odd = (float)(sigma * z1);
}

// y = w with the noise added inside the ranges; n elements, a multiple of 4.  VEC: both pointers 16-byte aligned.
template <bool VEC>
__global__ void __launch_bounds__(WN_THREADS)
weight_noise_kernel(const float *__restrict__ w, float *__restrict__ y, int64_t n, const __grid_constant__ NoiseRanges r,
                    double sigma, uint2 key, const int64_t *__restrict__ step) {
    const uint32_t s32 = (uint32_t)(*step);
    const int64_t nq = n / 4;
    int k = 0;      // the first range that does not end at or before this thread's quad
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e0 = 4 * q;
        while (k < r.n && r.hi[k] <= e0) ++k;
        float4 v;
        if (VEC) {
            v = __ldg(reinterpret_cast<const float4 *>(w) + q);
        } else {
            v = make_float4(__ldg(w + e0), __ldg(w + e0 + 1), __ldg(w + e0 + 2), __ldg(w + e0 + 3));
        }
        if (k < r.n && r.lo[k] < e0 + 4) {      // lo is a multiple of 4: the quad starts inside the range
            const int64_t m = r.hi[k] - e0;     // its first m elements (at least 1) are noised
            const uint4 c = curand_Philox4x32_10(make_uint4(s32, (uint32_t)q, 1u, 0u), key);
            float z0, z1, z2, z3;
            box_muller(c.x, c.y, sigma, z0, z1);
            box_muller(c.z, c.w, sigma, z2, z3);
            v.x += z0;
            if (m > 1) v.y += z1;
            if (m > 2) v.z += z2;
            if (m > 3) v.w += z3;
        }
        if (VEC) {
            reinterpret_cast<float4 *>(y)[q] = v;
        } else {
            y[e0] = v.x;
            y[e0 + 1] = v.y;
            y[e0 + 2] = v.z;
            y[e0 + 3] = v.w;
        }
    }
}
}  // namespace

// The pass: y = w (n floats, a multiple of 4) with sigma * z added to the nr ranges [lo[i], hi[i]) (ascending, each lo a
// multiple of 4).  `step` is read on the device when the kernel runs.
int run_weight_noise(const float *w, float *y, int64_t n, const int64_t *lo, const int64_t *hi, int nr, float sigma,
                     uint64_t seed, const int64_t *step, cudaStream_t st) {
    if (nr > WN_MAX_RANGES || n % 4 != 0)
        return set_error(CTCB_EINVAL, "weight noise: %d ranges (at most %d) over %lld floats (a multiple of 4)", nr,
                         WN_MAX_RANGES, (long long)n);
    if (n == 0) return CTCB_OK;
    NoiseRanges r{};
    r.n = nr;
    for (int i = 0; i < nr; ++i) {
        r.lo[i] = lo[i];
        r.hi[i] = hi[i];
    }
    const int64_t want = (n / 4 + WN_THREADS - 1) / WN_THREADS;
    const int64_t cap = (int64_t)num_sms() * 16;        // grid-stride beyond ~16 blocks per SM
    const unsigned blocks = (unsigned)(want < cap ? want : cap);
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const bool vec = ((uintptr_t)w % 16) == 0 && ((uintptr_t)y % 16) == 0;
    if (vec)
        weight_noise_kernel<true><<<blocks, WN_THREADS, 0, st>>>(w, y, n, r, (double)sigma, key, step);
    else
        weight_noise_kernel<false><<<blocks, WN_THREADS, 0, st>>>(w, y, n, r, (double)sigma, key, step);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb
