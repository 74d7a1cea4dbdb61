// subsample.cu -- frame stacking below a reduced-rate layer (include/ctcb200.h: subsample), forward and backward.
//
// Both kernels permute between the time-major layouts [T][B][n] = [T'][k][B][n] (k sub-frames of n units) and
// [T'][B][k n], T' = ceil(T / k):
//   stack   : S[t'][u][m n + j] = X[k t' + m][u][j], or 0 where k t' + m >= min(T_u, Tmax)
//   unstack : D[t][u][j] = dS[t / k][u][(t % k) n + j] for t < T_u, else 0
// They are exact copies (no arithmetic), so their bits do not depend on the launch shape.  Work is cut into n-float
// "sub-rows": one of the k pieces of a stacked row, which is one row of the full-rate side.  A block holds ty
// sub-rows of tx threads each; a thread copies every tx-th group of its sub-row, 16 bytes at a time where n % 4 == 0
// and every pointer is 16-byte aligned, else one float.
#include "common.cuh"

namespace ctcb {

namespace {
template <typename V>
__device__ __forceinline__ V zero_v();
template <> __device__ __forceinline__ float zero_v<float>() { return 0.f; }
template <> __device__ __forceinline__ float4 zero_v<float4>() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// nv groups of V per sub-row; sub-row s = (t' B + u) k + m of S, which is row (k t' + m) B + u of X
template <typename V>
__global__ void stack_kernel(const V *__restrict__ X, const int32_t *__restrict__ Tlen, int Tmax, int B, int nv, int k,
                             int nsub, V *__restrict__ S, int32_t *__restrict__ lens_out) {
    if (lens_out && blockIdx.x == 0 && threadIdx.y == 0)
        for (int u = threadIdx.x; u < B; u += blockDim.x) {
            int T = Tlen[u];
            T = T < 0 ? 0 : (T > Tmax ? Tmax : T);
            lens_out[u] = (T + k - 1) / k;
        }
    for (int64_t s64 = (int64_t)blockIdx.x * blockDim.y + threadIdx.y; s64 < nsub; s64 += (int64_t)gridDim.x * blockDim.y) {
        const int s = (int)s64;     // < nsub <= 2^31 - 1
        const int m = s % k, q = s / k;
        const int u = q % B, tp = q / B;
        const int t = tp * k + m;
        const bool valid = t < Tmax && t < Tlen[u];
        V *dst = S + (int64_t)s * nv;
        const V *src = X + ((int64_t)t * B + u) * nv;
        for (int j = threadIdx.x; j < nv; j += blockDim.x) dst[j] = valid ? src[j] : zero_v<V>();
    }
}

// sub-row r = t B + u of D, which is sub-row ((t / k) B + u) k + t % k of dS
template <typename V>
__global__ void unstack_kernel(const V *__restrict__ dS, const int32_t *__restrict__ Tlen, int B, int nv, int k,
                               int nsub, V *__restrict__ D) {
    for (int64_t r64 = (int64_t)blockIdx.x * blockDim.y + threadIdx.y; r64 < nsub; r64 += (int64_t)gridDim.x * blockDim.y) {
        const int r = (int)r64;     // < nsub <= 2^31 - 1
        const int t = r / B, u = r % B;
        const bool valid = t < Tlen[u];
        V *dst = D + (int64_t)r * nv;
        const V *src = dS + ((int64_t)((t / k) * B + u) * k + t % k) * nv;
        for (int j = threadIdx.x; j < nv; j += blockDim.x) dst[j] = valid ? src[j] : zero_v<V>();
    }
}

// tx threads per sub-row (a multiple of 32, at most 256), ty = 256 / tx sub-rows per block, grid-stride beyond ~16
// blocks per SM
struct CopyShape {
    dim3 block;
    unsigned grid;
};
CopyShape copy_shape(int nv, int nsub) {
    int tx = (nv + 31) / 32 * 32;
    if (tx > 256) tx = 256;
    const int ty = 256 / tx;
    const int64_t want = ((int64_t)nsub + ty - 1) / ty;
    const int64_t cap = (int64_t)num_sms() * 16;
    return {dim3(tx, ty), (unsigned)(want < cap ? (want > 0 ? want : 1) : cap)};
}

bool vec_ok(int n, const void *a, const void *b) { return n % 4 == 0 && ((((uintptr_t)a) | ((uintptr_t)b)) & 15) == 0; }
}  // namespace

int64_t subsampled_frames(int T, int k) { return k > 1 ? ((int64_t)T + k - 1) / k : T; }

int run_frame_stack(const float *x, const int32_t *Tlen, int Tmax, int B, int n, int k, float *s_out, int32_t *lens_out,
                    cudaStream_t st) {
    const int Tp = (int)subsampled_frames(Tmax, k);
    const int nsub = Tp * B * k;
    if (vec_ok(n, x, s_out)) {
        const CopyShape c = copy_shape(n / 4, nsub);
        stack_kernel<float4><<<c.grid, c.block, 0, st>>>((const float4 *)x, Tlen, Tmax, B, n / 4, k, nsub,
                                                         (float4 *)s_out, lens_out);
    } else {
        const CopyShape c = copy_shape(n, nsub);
        stack_kernel<float><<<c.grid, c.block, 0, st>>>(x, Tlen, Tmax, B, n, k, nsub, s_out, lens_out);
    }
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

int run_frame_unstack(const float *ds, const int32_t *Tlen, int Tmax, int B, int n, int k, float *d_out, cudaStream_t st) {
    const int nsub = Tmax * B;
    if (vec_ok(n, ds, d_out)) {
        const CopyShape c = copy_shape(n / 4, nsub);
        unstack_kernel<float4><<<c.grid, c.block, 0, st>>>((const float4 *)ds, Tlen, B, n / 4, k, nsub, (float4 *)d_out);
    } else {
        const CopyShape c = copy_shape(n, nsub);
        unstack_kernel<float><<<c.grid, c.block, 0, st>>>(ds, Tlen, B, n, k, nsub, d_out);
    }
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb

using namespace ctcb;

static int stack_check(const char *fn, int Tmax, int B, int n, int k) {
    if (Tmax <= 0 || B <= 0 || n <= 0 || k < 1 || (int64_t)subsampled_frames(Tmax, k) * B * k > 0x7fffffff ||
        (int64_t)Tmax * B > 0x7fffffff)
        return set_error(CTCB_EINVAL, "%s: Tmax = %d, B = %d, n = %d, k = %d (need all >= 1 and ceil(Tmax / k) * k * B "
                         "< 2^31)", fn, Tmax, B, n, k);
    return CTCB_OK;
}

extern "C" int ctcb_frame_stack_f32(const float *x, const int32_t *T_per_utt, int Tmax, int B, int n, int k,
                                    float *s_out, int32_t *lens_out, void *stream) {
    if (int rc = stack_check("ctcb_frame_stack_f32", Tmax, B, n, k)) return rc;
    if (!x || !T_per_utt || !s_out) return set_error(CTCB_EINVAL, "ctcb_frame_stack_f32: null pointer argument");
    return run_frame_stack(x, T_per_utt, Tmax, B, n, k, s_out, lens_out, (cudaStream_t)stream);
}

extern "C" int ctcb_frame_unstack_f32(const float *ds, const int32_t *T_per_utt, int Tmax, int B, int n, int k,
                                      float *d_out, void *stream) {
    if (int rc = stack_check("ctcb_frame_unstack_f32", Tmax, B, n, k)) return rc;
    if (!ds || !T_per_utt || !d_out) return set_error(CTCB_EINVAL, "ctcb_frame_unstack_f32: null pointer argument");
    return run_frame_unstack(ds, T_per_utt, Tmax, B, n, k, d_out, (cudaStream_t)stream);
}
