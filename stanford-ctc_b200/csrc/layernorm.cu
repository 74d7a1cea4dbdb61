// layernorm.cu -- layer normalisation of a ReLU hidden layer (include/ctcb200.h: layerNorm), forward and backward.
//
// Rows are time-major [R][H] fp32 frames.  One CTA works on one row at a time; thread t owns the units
// t + k * blockDim.x (k < NPT) of every row it sees (groups of four units, one float4, when H % 4 == 0), so a row is
// read once into registers and the per-unit parameters and parameter-gradient partials stay in registers too.  Row
// sums go through warp_sum and then the warps' totals in warp order: the bits depend only on H and the launch shape,
// which depends only on H.
//
//   forward : mu = mean z, var = mean (z - mu)^2 (two passes over the registers), rstd = 1 / sqrt(var + eps),
//             y = relu(gamma * (z - mu) * rstd + beta); y may alias z.  mu / rstd are written when given.
//   backward: in place on the delta d, g on entry: xh recomputed as the forward computed it, gh = g gamma,
//             dz = rstd (gh - mean gh - xh mean(gh xh)); CTA b sums g xh and g over its fixed chunk of rows into
//             partial[0][b][:] and partial[1][b][:], and a second launch adds the chunks in block order.
#include "common.cuh"

namespace ctcb {

namespace {
constexpr float LN_EPS = 1e-5f;
constexpr int LN_MAX_PARTS = 1024;      // CTAs (row chunks) of the backward pass, so rows of its partial area
constexpr int LN_MIN_ROWS = 8;          // rows per chunk at least

// The launch shape for width H: threads per CTA and the slots (units, or float4 groups) per thread.
struct LnShape {
    bool vec;
    int threads, npt;
};
LnShape ln_shape(int H) {
    LnShape s;
    s.vec = (H % 4 == 0);
    const int Q = (H + 3) / 4;                             // slots per row
    int t = ((Q + 1) / 2 + 31) / 32 * 32;                  // two slots per thread where 256 threads allow it
    if (t > 256) t = 256;
    const int need = (Q + t - 1) / t;                      // <= 8 for H <= CTCB_LAYERNORM_MAX_H
    s.threads = t;
    s.npt = need <= 1 ? 1 : need <= 2 ? 2 : need <= 4 ? 4 : 8;
    return s;
}
int64_t ln_parts(int64_t R) {
    int64_t rpb = (R + LN_MAX_PARTS - 1) / LN_MAX_PARTS;
    if (rpb < LN_MIN_ROWS) rpb = LN_MIN_ROWS;
    return rpb;
}

// The sum of v over the CTA, the same value in every thread; red: 32 floats of shared memory.
__device__ __forceinline__ float block_sum(float v, float *red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    __syncthreads();
    return t;
}
__device__ __forceinline__ float2 block_sum2(float a, float b, float2 *red) {
    a = warp_sum(a);
    b = warp_sum(b);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = make_float2(a, b);
    __syncthreads();
    float2 t = make_float2(0.f, 0.f);
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
        t.x += red[i].x;
        t.y += red[i].y;
    }
    __syncthreads();
    return t;
}

// Slot k of thread t: units 4q .. 4q+3, q = t + k * blockDim.x; one float4 (VEC: H % 4 == 0, so every row starts
// 16-byte aligned) or scalar accesses, the units past the row reading 0 and never written.
template <bool VEC>
__device__ __forceinline__ int slot_units(int q, int H) {
    const int n = H - 4 * q;
    return n <= 0 ? 0 : n >= 4 ? 4 : n;
}
template <bool VEC>
__device__ __forceinline__ float4 load_slot(const float *row, int q, int H) {
    if (VEC) return 4 * q < H ? reinterpret_cast<const float4 *>(row)[q] : make_float4(0.f, 0.f, 0.f, 0.f);
    const int n = slot_units<VEC>(q, H);
    const float *p = row + 4 * q;
    return make_float4(n > 0 ? p[0] : 0.f, n > 1 ? p[1] : 0.f, n > 2 ? p[2] : 0.f, n > 3 ? p[3] : 0.f);
}
template <bool VEC>
__device__ __forceinline__ void store_slot(float *row, int q, int H, float4 v) {
    if (VEC) {
        if (4 * q < H) reinterpret_cast<float4 *>(row)[q] = v;
        return;
    }
    const int n = slot_units<VEC>(q, H);
    float *p = row + 4 * q;
    if (n > 0) p[0] = v.x;
    if (n > 1) p[1] = v.y;
    if (n > 2) p[2] = v.z;
    if (n > 3) p[3] = v.w;
}

__device__ __forceinline__ float get(const float4 &v, int c) { return c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w; }
__device__ __forceinline__ void put(float4 &v, int c, float x) {
    if (c == 0) v.x = x; else if (c == 1) v.y = x; else if (c == 2) v.z = x; else v.w = x;
}

template <bool VEC, int NPT>
__global__ void __launch_bounds__(256) ln_forward_kernel(const float *z, float *y, float *__restrict__ mu_out,
                                                          float *__restrict__ rstd_out, const float *__restrict__ gamma,
                                                          const float *__restrict__ beta, int64_t R, int H) {
    __shared__ float red[32];
    float4 ga[NPT], be[NPT];
#pragma unroll
    for (int k = 0; k < NPT; ++k) {
        const int q = threadIdx.x + k * blockDim.x;
        ga[k] = load_slot<VEC>(gamma, q, H);
        be[k] = load_slot<VEC>(beta, q, H);
    }
    const float fH = (float)H;
    for (int64_t r = blockIdx.x; r < R; r += gridDim.x) {
        const float *zr = z + r * H;
        float4 v[NPT];
#pragma unroll
        for (int k = 0; k < NPT; ++k) v[k] = load_slot<VEC>(zr, threadIdx.x + k * blockDim.x, H);
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < NPT; ++k) s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
        const float mu = block_sum(s, red) / fH;
        float ss = 0.f;
#pragma unroll
        for (int k = 0; k < NPT; ++k) {
            const int n = slot_units<VEC>(threadIdx.x + k * blockDim.x, H);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float d = c < n ? get(v[k], c) - mu : 0.f;
                ss = fmaf(d, d, ss);
            }
        }
        const float var = block_sum(ss, red) / fH;
        const float rstd = 1.f / sqrtf(var + LN_EPS);
        if (mu_out && threadIdx.x == 0) {
            mu_out[r] = mu;
            rstd_out[r] = rstd;
        }
        float *yr = y + r * H;
#pragma unroll
        for (int k = 0; k < NPT; ++k) {
            float4 o;
#pragma unroll
            for (int c = 0; c < 4; ++c) put(o, c, fmaxf(fmaf(get(ga[k], c), (get(v[k], c) - mu) * rstd, get(be[k], c)), 0.f));
            store_slot<VEC>(yr, threadIdx.x + k * blockDim.x, H, o);
        }
    }
}

template <bool VEC, int NPT>
__global__ void __launch_bounds__(256) ln_backward_kernel(float *__restrict__ d, const float *__restrict__ z,
                                                           const float *__restrict__ mu, const float *__restrict__ rstd,
                                                           const float *__restrict__ gamma, int64_t R, int H,
                                                           int64_t rows_per_part, float *__restrict__ partial) {
    __shared__ float2 red[32];
    float4 ga[NPT], ag[NPT], ab[NPT];
#pragma unroll
    for (int k = 0; k < NPT; ++k) {
        ga[k] = load_slot<VEC>(gamma, threadIdx.x + k * blockDim.x, H);
        ag[k] = ab[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float fH = (float)H;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_part;
    const int64_t r1 = (r0 + rows_per_part < R) ? r0 + rows_per_part : R;
    for (int64_t r = r0; r < r1; ++r) {
        const float m = mu[r], rs = rstd[r];
        float4 g[NPT], xh[NPT];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int k = 0; k < NPT; ++k) {
            const int q = threadIdx.x + k * blockDim.x;
            g[k] = load_slot<VEC>(d + r * H, q, H);
            const float4 zz = load_slot<VEC>(z + r * H, q, H);
            const int n = slot_units<VEC>(q, H);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float x = c < n ? (get(zz, c) - m) * rs : 0.f;     // the forward's xh, bit for bit
                put(xh[k], c, x);
                const float gh = get(g[k], c) * get(ga[k], c);
                s1 += gh;
                s2 = fmaf(gh, x, s2);
            }
        }
        const float2 t = block_sum2(s1, s2, red);
        const float a = t.x / fH, b = t.y / fH;
#pragma unroll
        for (int k = 0; k < NPT; ++k) {
            float4 o;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float gg = get(g[k], c), x = get(xh[k], c);
                // + 0: a zero row of g (a padded frame) gives +0.0, where a negative gamma would leave -0.0
                put(o, c, rs * (gg * get(ga[k], c) - a - x * b) + 0.f);
                put(ag[k], c, fmaf(gg, x, get(ag[k], c)));
                put(ab[k], c, get(ab[k], c) + gg);
            }
            store_slot<VEC>(d + r * H, threadIdx.x + k * blockDim.x, H, o);
        }
    }
    float *pg = partial + (int64_t)blockIdx.x * H;
    float *pb = partial + ((int64_t)gridDim.x + blockIdx.x) * H;
#pragma unroll
    for (int k = 0; k < NPT; ++k) {
        store_slot<VEC>(pg, threadIdx.x + k * blockDim.x, H, ag[k]);
        store_slot<VEC>(pb, threadIdx.x + k * blockDim.x, H, ab[k]);
    }
}

// dgamma (blockIdx.y = 0) and dbeta (1): unit n sums the partial rows of the parts in a fixed order, eight strided
// streams and then the eight in order.  ACC: add into out (a later micro-batch of the step).
template <bool ACC>
__global__ void ln_param_grad_kernel(const float *__restrict__ partial, int parts, int H, float *__restrict__ dgamma,
                                     float *__restrict__ dbeta) {
    __shared__ float sh[8][33];
    const int n = blockIdx.x * 32 + threadIdx.x;
    const float *p = partial + (int64_t)blockIdx.y * parts * H;
    float s = 0.f;
    if (n < H)
        for (int i = threadIdx.y; i < parts; i += 8) s += p[(int64_t)i * H + n];
    sh[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && n < H) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sh[i][threadIdx.x];
        float *out = blockIdx.y ? dbeta : dgamma;
        if (ACC) t += out[n];
        out[n] = t;
    }
}

template <int NPT>
void launch_forward(const LnShape &s, unsigned grid, const float *z, float *y, float *mu, float *rstd,
                    const float *gamma, const float *beta, int64_t R, int H, cudaStream_t st) {
    if (s.vec) ln_forward_kernel<true, NPT><<<grid, s.threads, 0, st>>>(z, y, mu, rstd, gamma, beta, R, H);
    else ln_forward_kernel<false, NPT><<<grid, s.threads, 0, st>>>(z, y, mu, rstd, gamma, beta, R, H);
}
template <int NPT>
void launch_backward(const LnShape &s, unsigned grid, float *d, const float *z, const float *mu, const float *rstd,
                     const float *gamma, int64_t R, int H, int64_t rpp, float *partial, cudaStream_t st) {
    if (s.vec) ln_backward_kernel<true, NPT><<<grid, s.threads, 0, st>>>(d, z, mu, rstd, gamma, R, H, rpp, partial);
    else ln_backward_kernel<false, NPT><<<grid, s.threads, 0, st>>>(d, z, mu, rstd, gamma, R, H, rpp, partial);
}
}  // namespace

size_t layernorm_workspace_bytes(int64_t R, int H) {
    if (R <= 0 || H <= 0) return 0;
    const int64_t parts = (R + LN_MIN_ROWS - 1) / LN_MIN_ROWS < LN_MAX_PARTS ? (R + LN_MIN_ROWS - 1) / LN_MIN_ROWS
                                                                             : LN_MAX_PARTS;
    return align_up((size_t)2 * parts * H * sizeof(float), 256);
}

int run_layernorm_forward(const float *z, float *y, float *mu, float *rstd, const float *gamma, const float *beta,
                          int64_t R, int H, cudaStream_t st) {
    if (R <= 0) return CTCB_OK;
    const LnShape s = ln_shape(H);
    const int64_t cap = (int64_t)num_sms() * (2048 / s.threads);      // one resident wave, each CTA strides rows
    const unsigned grid = (unsigned)(R < cap ? R : cap);
    switch (s.npt) {
    case 1: launch_forward<1>(s, grid, z, y, mu, rstd, gamma, beta, R, H, st); break;
    case 2: launch_forward<2>(s, grid, z, y, mu, rstd, gamma, beta, R, H, st); break;
    case 4: launch_forward<4>(s, grid, z, y, mu, rstd, gamma, beta, R, H, st); break;
    default: launch_forward<8>(s, grid, z, y, mu, rstd, gamma, beta, R, H, st); break;
    }
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

int run_layernorm_backward(float *d, const float *z, const float *mu, const float *rstd, const float *gamma,
                           float *dgamma, float *dbeta, int64_t R, int H, bool accumulate, float *partial,
                           cudaStream_t st) {
    if (R <= 0) return CTCB_OK;
    const LnShape s = ln_shape(H);
    const int64_t rpp = ln_parts(R);
    const int parts = (int)((R + rpp - 1) / rpp);
    switch (s.npt) {
    case 1: launch_backward<1>(s, parts, d, z, mu, rstd, gamma, R, H, rpp, partial, st); break;
    case 2: launch_backward<2>(s, parts, d, z, mu, rstd, gamma, R, H, rpp, partial, st); break;
    case 4: launch_backward<4>(s, parts, d, z, mu, rstd, gamma, R, H, rpp, partial, st); break;
    default: launch_backward<8>(s, parts, d, z, mu, rstd, gamma, R, H, rpp, partial, st); break;
    }
    CTCB_LAUNCH_CHECK();
    const dim3 grid((H + 31) / 32, 2);
    if (accumulate) ln_param_grad_kernel<true><<<grid, dim3(32, 8), 0, st>>>(partial, parts, H, dgamma, dbeta);
    else ln_param_grad_kernel<false><<<grid, dim3(32, 8), 0, st>>>(partial, parts, H, dgamma, dbeta);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb

using namespace ctcb;

extern "C" size_t ctcb_layernorm_workspace_bytes(int64_t R, int H) {
    return (H > CTCB_LAYERNORM_MAX_H) ? 0 : layernorm_workspace_bytes(R, H);
}

static int ln_check(const char *fn, int64_t R, int H) {
    if (R < 0 || H <= 0 || H > CTCB_LAYERNORM_MAX_H)
        return set_error(CTCB_EINVAL, "%s: R = %lld, H = %d (need R >= 0, 1 <= H <= %d)", fn, (long long)R, H,
                         CTCB_LAYERNORM_MAX_H);
    return CTCB_OK;
}

extern "C" int ctcb_layernorm_forward_f32(const float *z, float *y, float *mu, float *rstd, const float *gamma,
                                          const float *beta, int64_t R, int H, void *stream) {
    if (int rc = ln_check("ctcb_layernorm_forward_f32", R, H)) return rc;
    if (!z || !y || !gamma || !beta || (!mu) != (!rstd))
        return set_error(CTCB_EINVAL, "ctcb_layernorm_forward_f32: null pointer argument (mu and rstd: both or neither)");
    if (H % 4 == 0 && ((((uintptr_t)z) | ((uintptr_t)y) | ((uintptr_t)gamma) | ((uintptr_t)beta)) & 15))
        return set_error(CTCB_EINVAL, "ctcb_layernorm_forward_f32: H %% 4 == 0 needs 16-byte aligned z, y, gamma, beta");
    return run_layernorm_forward(z, y, mu, rstd, gamma, beta, R, H, (cudaStream_t)stream);
}

extern "C" int ctcb_layernorm_backward_f32(float *delta, const float *z, const float *mu, const float *rstd,
                                           const float *gamma, float *dgamma, float *dbeta, int64_t R, int H,
                                           int accumulate, void *workspace, size_t ws_bytes, void *stream) {
    if (int rc = ln_check("ctcb_layernorm_backward_f32", R, H)) return rc;
    if (!delta || !z || !mu || !rstd || !gamma || !dgamma || !dbeta || !workspace)
        return set_error(CTCB_EINVAL, "ctcb_layernorm_backward_f32: null pointer argument");
    if (H % 4 == 0 && ((((uintptr_t)delta) | ((uintptr_t)z) | ((uintptr_t)gamma) | ((uintptr_t)workspace)) & 15))
        return set_error(CTCB_EINVAL, "ctcb_layernorm_backward_f32: H %% 4 == 0 needs 16-byte aligned delta, z, gamma "
                         "and workspace");
    const size_t need = layernorm_workspace_bytes(R, H);
    if (ws_bytes < need)
        return set_error(CTCB_ENOMEM, "ctcb_layernorm_backward_f32: workspace %zu < %zu bytes", ws_bytes, need);
    return run_layernorm_backward(delta, z, mu, rstd, gamma, dgamma, dbeta, R, H, accumulate != 0, (float *)workspace,
                                  (cudaStream_t)stream);
}
