// input_mask.cu -- SpecAugment frequency and time masks of the input features: one pass that copies the time-major
// features [Tmax][B][inputDim] and writes +0 over the masked bands, and the checks of its layout and policy.
//
// The policy is defined once, at ctcb_brnn_set_input_masks in include/ctcb200.h (the tests restate it in NumPy): mask k
// of minibatch utterance g at optimisation step s draws (r0, r1, r2, r3) = Philox4x32-10(counter = (s mod 2^32,
// g mod 2^32, 0, k), key = (seed mod 2^32, seed >> 32)); masks k < mF are bands of filter-bank bins, the others spans
// of raw frames.  Row t' of utterance u holds c = inputDim / nu frame slots of nu bins, slot j the raw frame
// clamp(t' + j - h, 0, T_u - 1), h = (c - 1) / 2.
//
// One CTA takes `rows` consecutive frames of one utterance.  It draws that utterance's bands first (one thread per
// mask) and turns them into two bit sets in shared memory: the masked bins, and the masked raw frames its rows can
// reach.  Every element then costs two shared-memory bit tests next to its load and store.
#include "common.cuh"
#include <curand_philox4x32_x.h>

namespace ctcb {

namespace {
constexpr int MASK_THREADS = 256;
constexpr int MASK_MAX = 64;                    // masks of each kind
constexpr int MASK_ELEMS = 8192;                // elements per CTA: rows = clamp(MASK_ELEMS / inputDim, 1, 64)
constexpr size_t MASK_SMEM_MAX = 48 * 1024;     // the bit sets stay within the default dynamic shared memory

int mask_rows(int D) {
    const int r = MASK_ELEMS / D;
    return r < 1 ? 1 : r > 64 ? 64 : r;
}
// words of the two bit sets: nu bins, and the raw frames rows t'..t'+rows-1 reach (rows + 2h of them)
size_t mask_smem_bytes(int D, int nu) {
    const int64_t c = D / nu;
    return sizeof(uint32_t) * (size_t)(((int64_t)nu + 31) / 32 + ((int64_t)mask_rows(D) + c - 1 + 31) / 32);
}

__device__ __forceinline__ bool bit(const uint32_t *bits, int i) { return (bits[i >> 5] >> (i & 31)) & 1u; }

// x, y: [Tmax][B][D], y = x with the masked elements +0.  VEC: D % 4 == 0 and both 16-byte aligned.
template <bool VEC>
__global__ void __launch_bounds__(MASK_THREADS)
input_mask_kernel(const float *__restrict__ x, float *__restrict__ y, const int32_t *__restrict__ lens, int B, int Tmax,
                  int D, int nu, int h, int rows, int mF, int F, int mT, int Tw, double p, uint2 key,
                  const int64_t *__restrict__ step, int64_t first, int64_t stride) {
    extern __shared__ uint32_t bits[];          // [nF] masked bins, then the masked raw frames lo..hi
    __shared__ int2 band[2 * MASK_MAX];         // [start, end) of every mask
    const int u = (int)(blockIdx.x % (unsigned)B);
    const int ta = (int)(blockIdx.x / (unsigned)B) * rows;
    const int tb = min(ta + rows, Tmax);
    const int Tu = lens[u];
    const int nF = (nu + 31) >> 5;
    // the raw frames slots of rows ta..min(tb, Tu) - 1 hold
    const int lo = max(ta - h, 0), hi = min(tb - 1 + h, Tu - 1);
    const bool masked = ta < Tu && mF + mT > 0;     // uniform over the CTA
    if (masked) {
        const int k = threadIdx.x;
        if (k < mF + mT) {
            const int64_t g = first + stride * (int64_t)u;
            const uint4 r = curand_Philox4x32_10(make_uint4((uint32_t)(*step), (uint32_t)g, 0u, (uint32_t)k), key);
            int a, w;
            if (k < mF) {
                w = (int)(((uint64_t)r.x * (uint64_t)(F + 1)) >> 32);
                a = (int)(((uint64_t)r.y * (uint64_t)(nu - w + 1)) >> 32);
            } else {
                const double pt = floor(p * (double)Tu);
                const int W = pt < (double)Tw ? (int)pt : Tw;
                w = (int)(((uint64_t)r.x * (uint64_t)(W + 1)) >> 32);
                a = (int)(((uint64_t)r.y * (uint64_t)(Tu - w + 1)) >> 32);
            }
            band[k] = make_int2(a, a + w);
        }
        __syncthreads();
        const int nT = (hi - lo + 1 + 31) >> 5;
        for (int wd = threadIdx.x; wd < nF + nT; wd += blockDim.x) {
            const bool freq = wd < nF;
            const int base = freq ? 32 * wd : lo + 32 * (wd - nF);
            uint32_t word = 0;
            for (int k = freq ? 0 : mF; k < (freq ? mF : mF + mT); ++k) {
                const int a = max(band[k].x - base, 0), b = min(band[k].y - base, 32);
                if (a < b) word |= (b - a == 32) ? 0xffffffffu : ((1u << (b - a)) - 1u) << a;
            }
            bits[wd] = word;
        }
        __syncthreads();
    }
    const uint32_t *tbits = bits + nF;
    const int Q = VEC ? D / 4 : D;
    const int n = (tb - ta) * Q;
#pragma unroll 4
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
        const int rr = idx / Q, q = idx - rr * Q;
        const int t = ta + rr;
        const int64_t off = ((int64_t)t * B + u) * D;
        if (VEC) {
            float4 v = __ldg(reinterpret_cast<const float4 *>(x + off) + q);
            if (masked && t < Tu) {
                int j = (4 * q) / nu, b = 4 * q - j * nu;
                float *e = &v.x;
#pragma unroll
                for (int s = 0; s < 4; ++s) {
                    const int f = min(max(t + j - h, 0), Tu - 1);
                    if (bit(bits, b) || bit(tbits, f - lo)) e[s] = 0.f;
                    if (++b == nu) b = 0, ++j;
                }
            }
            reinterpret_cast<float4 *>(y + off)[q] = v;
        } else {
            float v = __ldg(x + off + q);
            if (masked && t < Tu) {
                const int j = q / nu, b = q - j * nu;
                const int f = min(max(t + j - h, 0), Tu - 1);
                if (bit(bits, b) || bit(tbits, f - lo)) v = 0.f;
            }
            y[off + q] = v;
        }
    }
}
}  // namespace

// Why nu = featDim cannot lay out rows of D = inputDim features, or null.
const char *input_mask_layout_error(int D, int nu, char (&buf)[192]) {
    if (nu < 1 || D < 1 || D % nu != 0) {
        snprintf(buf, sizeof(buf), "featDim %d does not divide inputDim %d into whole frames", nu, D);
        return buf;
    }
    if ((D / nu) % 2 == 0) {
        snprintf(buf, sizeof(buf), "inputDim %d / featDim %d = %d frame slots: a spliced context is odd", D, nu, D / nu);
        return buf;
    }
    if (mask_smem_bytes(D, nu) > MASK_SMEM_MAX) {
        snprintf(buf, sizeof(buf), "inputDim %d with featDim %d: the mask pass's bit sets exceed %zu bytes", D, nu,
                 MASK_SMEM_MAX);
        return buf;
    }
    return nullptr;
}

// Why a policy is outside the limits of include/ctcb200.h, or null.  nu = 0: a net without a layout, which takes no
// mask.
const char *input_mask_policy_error(int nu, int mF, int F, int mT, int Tw, double p, char (&buf)[192]) {
    auto say = [&buf](const char *fmt, auto... args) -> const char * {
        snprintf(buf, sizeof(buf), fmt, args...);
        return buf;
    };
    if (mF < 0 || mF > MASK_MAX || mT < 0 || mT > MASK_MAX)
        return say("freqMasks %d and timeMasks %d must each be in 0..%d", mF, mT, MASK_MAX);
    if (F < 0 || (nu > 0 && F > nu)) return say("freqWidth %d is not in 0..featDim (%d)", F, nu);
    if (Tw < 0) return say("timeWidth %d is negative", Tw);
    if (!(p >= 0.0 && p <= 1.0)) return say("timeRatio %g is not in [0, 1]", p);
    if (mF + mT > 0 && nu == 0)
        return say("%d frequency and %d time masks need a feature layout (maskFeatDim > 0 in the config)", mF, mT);
    return nullptr;
}

int run_input_mask(const float *x, const int32_t *lens, int B, int Tmax, int D, int nu, int mF, int F, int mT, int Tw,
                   double p, uint64_t seed, const int64_t *step, int64_t first, int64_t stride, float *y,
                   cudaStream_t st) {
    const int rows = mask_rows(D);
    const int64_t blocks = (int64_t)B * ((Tmax + rows - 1) / rows);
    const size_t smem = mask_smem_bytes(D, nu);
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const int h = (D / nu - 1) / 2;
    const bool vec = D % 4 == 0 && ((uintptr_t)x % 16) == 0 && ((uintptr_t)y % 16) == 0;
    if (vec)
        input_mask_kernel<true><<<(unsigned)blocks, MASK_THREADS, smem, st>>>(x, y, lens, B, Tmax, D, nu, h, rows, mF, F,
                                                                              mT, Tw, p, key, step, first, stride);
    else
        input_mask_kernel<false><<<(unsigned)blocks, MASK_THREADS, smem, st>>>(x, y, lens, B, Tmax, D, nu, h, rows, mF,
                                                                               F, mT, Tw, p, key, step, first, stride);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb

extern "C" int ctcb_input_mask_f32(const float *feats, const int32_t *T_per_utt, int B, int Tmax, int inputDim,
                                   int featDim, int freqMasks, int freqWidth, int timeMasks, int timeWidth,
                                   double timeRatio, uint64_t seed, const int64_t *step, int64_t first, int64_t stride,
                                   float *out, void *stream) {
    char buf[192];
    if (!feats || !T_per_utt || !out || (freqMasks + timeMasks > 0 && !step))
        return ctcb::set_error(CTCB_EINVAL, "ctcb_input_mask_f32: null pointer argument");
    if (B < 1 || Tmax < 1 || (int64_t)B * Tmax > 0x7fffffff)
        return ctcb::set_error(CTCB_EINVAL, "ctcb_input_mask_f32: B = %d, Tmax = %d (need both >= 1, B * Tmax < 2^31)",
                               B, Tmax);
    if (const char *why = ctcb::input_mask_layout_error(inputDim, featDim, buf))
        return ctcb::set_error(CTCB_EINVAL, "ctcb_input_mask_f32: %s", why);
    if (const char *why = ctcb::input_mask_policy_error(featDim, freqMasks, freqWidth, timeMasks, timeWidth, timeRatio, buf))
        return ctcb::set_error(CTCB_EINVAL, "ctcb_input_mask_f32: %s", why);
    if (first < 0 || stride < 1)
        return ctcb::set_error(CTCB_EINVAL, "ctcb_input_mask_f32: first = %lld, stride = %lld (need first >= 0, stride >= 1)",
                               (long long)first, (long long)stride);
    return ctcb::run_input_mask(feats, T_per_utt, B, Tmax, inputDim, featDim, freqMasks, freqWidth, timeMasks, timeWidth,
                                timeRatio, seed, step, first, stride, out, (cudaStream_t)stream);
}
