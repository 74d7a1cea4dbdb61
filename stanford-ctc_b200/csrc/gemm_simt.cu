// gemm_simt.cu -- exact-fp32 dense contraction (FFMA), the arithmetic of the reference's
// cudamat `cm.dot` (legacy cuBLAS sgemm; call sites ctc_fast/nnets/brnnet.py:140,196,204,227-230).
//
// Row-major C[MxN] = alpha*op(A)*op(B) + beta*C with a fused epilogue (column bias, ReLU,
// sign-mask of another matrix).  128x128x16 tiles, 256 threads, 8x8 register micro-tiles,
// register-staged double buffering; split-K across gridDim.z for the weight-gradient shapes
// (M,N = layer sizes, K = all frames of the batch), reduced deterministically by a second kernel.
//
// This is the precision-exact path; the tensor-core path for the large contractions is gemm_tc.cu.
#include "common.cuh"

namespace ctcb {

constexpr int BM = 128, BN = 128, BK = 16, NT = 256;

struct GemmArgs {
    int M, N, K;
    const float *A; int64_t lda;
    const float *B; int64_t ldb;
    float *C; int64_t ldc;
    float alpha, beta;
    const float *bias; int relu; const float *mask;
    float *partial;   // split-K partials [splits][M][N] (nullptr when splits == 1)
    int k_per_split;
    int vecc;         // C (and mask / partial) rows are 16-byte aligned: the epilogue stores float4
};

__device__ __forceinline__ float epilogue(const GemmArgs &g, float acc, int m, int n) {
    float v = g.alpha * acc;
    if (g.beta != 0.f) v += g.beta * g.C[(int64_t)m * g.ldc + n];
    if (g.bias) v += g.bias[n];
    if (g.relu) v = fmaxf(v, 0.f);
    if (g.mask) v = (g.mask[(int64_t)m * g.ldc + n] > 0.f) ? v : 0.f;
    return v;
}

// the same on four consecutive columns (same operations in the same order: bit-identical to the scalar form)
__device__ __forceinline__ float4 epilogue4(const GemmArgs &g, float4 acc, int m, int n) {
    float4 v = make_float4(g.alpha * acc.x, g.alpha * acc.y, g.alpha * acc.z, g.alpha * acc.w);
    if (g.beta != 0.f) {
        const float4 c = *reinterpret_cast<const float4 *>(g.C + (int64_t)m * g.ldc + n);
        v.x += g.beta * c.x; v.y += g.beta * c.y; v.z += g.beta * c.z; v.w += g.beta * c.w;
    }
    if (g.bias) { v.x += g.bias[n]; v.y += g.bias[n + 1]; v.z += g.bias[n + 2]; v.w += g.bias[n + 3]; }
    if (g.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    if (g.mask) {
        const float4 k = *reinterpret_cast<const float4 *>(g.mask + (int64_t)m * g.ldc + n);
        v.x = (k.x > 0.f) ? v.x : 0.f; v.y = (k.y > 0.f) ? v.y : 0.f; v.z = (k.z > 0.f) ? v.z : 0.f; v.w = (k.w > 0.f) ? v.w : 0.f;
    }
    return v;
}

// TA: A stored K x M (reduction index is the row).  TB: B stored N x K.
template <bool TA, bool TB, bool VEC>
__global__ void __launch_bounds__(NT) gemm_simt_kernel(GemmArgs g) {
    __shared__ __align__(16) float As[2][BK][BM + 4];
    __shared__ __align__(16) float Bs[2][BK][BN + 4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int kbeg = blockIdx.z * g.k_per_split;
    const int kend = min(g.K, kbeg + g.k_per_split);
    const int tx = tid & 15, ty = tid >> 4;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    // global -> register staging: each thread moves 2 float4 (8 floats) of A and of B per k-tile
    float ra[8], rb[8];

    auto load_a = [&](int k0) {
        if (!TA) {  // A[m][k], k contiguous: 128 rows x 16 k -> 4 float4 per row
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int idx = tid + h * NT;           // 0..511
                const int r = idx >> 2, c4 = (idx & 3) * 4;
                const int m = m0 + r, k = k0 + c4;
                const float *p = g.A + (int64_t)m * g.lda + k;
                if (VEC && m < g.M && k + 3 < kend) {
                    const float4 v = *reinterpret_cast<const float4 *>(p);
                    ra[h * 4 + 0] = v.x; ra[h * 4 + 1] = v.y; ra[h * 4 + 2] = v.z; ra[h * 4 + 3] = v.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) ra[h * 4 + e] = (m < g.M && k + e < kend) ? p[e] : 0.f;
                }
            }
        } else {    // A[k][m], m contiguous: 16 k x 128 m -> 32 float4 per k row
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int idx = tid + h * NT;
                const int r = idx >> 5, c4 = (idx & 31) * 4;
                const int k = k0 + r, m = m0 + c4;
                const float *p = g.A + (int64_t)k * g.lda + m;
                if (VEC && k < kend && m + 3 < g.M) {
                    const float4 v = *reinterpret_cast<const float4 *>(p);
                    ra[h * 4 + 0] = v.x; ra[h * 4 + 1] = v.y; ra[h * 4 + 2] = v.z; ra[h * 4 + 3] = v.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) ra[h * 4 + e] = (k < kend && m + e < g.M) ? p[e] : 0.f;
                }
            }
        }
    };
    auto load_b = [&](int k0) {
        if (TB) {   // B[n][k], k contiguous
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int idx = tid + h * NT;
                const int r = idx >> 2, c4 = (idx & 3) * 4;
                const int n = n0 + r, k = k0 + c4;
                const float *p = g.B + (int64_t)n * g.ldb + k;
                if (VEC && n < g.N && k + 3 < kend) {
                    const float4 v = *reinterpret_cast<const float4 *>(p);
                    rb[h * 4 + 0] = v.x; rb[h * 4 + 1] = v.y; rb[h * 4 + 2] = v.z; rb[h * 4 + 3] = v.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) rb[h * 4 + e] = (n < g.N && k + e < kend) ? p[e] : 0.f;
                }
            }
        } else {    // B[k][n], n contiguous
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int idx = tid + h * NT;
                const int r = idx >> 5, c4 = (idx & 31) * 4;
                const int k = k0 + r, n = n0 + c4;
                const float *p = g.B + (int64_t)k * g.ldb + n;
                if (VEC && k < kend && n + 3 < g.N) {
                    const float4 v = *reinterpret_cast<const float4 *>(p);
                    rb[h * 4 + 0] = v.x; rb[h * 4 + 1] = v.y; rb[h * 4 + 2] = v.z; rb[h * 4 + 3] = v.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) rb[h * 4 + e] = (k < kend && n + e < g.N) ? p[e] : 0.f;
                }
            }
        }
    };
    auto store_a = [&](int buf) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int idx = tid + h * NT;
            if (!TA) {
                const int r = idx >> 2, c4 = (idx & 3) * 4;
#pragma unroll
                for (int e = 0; e < 4; ++e) As[buf][c4 + e][r] = ra[h * 4 + e];
            } else {
                const int r = idx >> 5, c4 = (idx & 31) * 4;
                *reinterpret_cast<float4 *>(&As[buf][r][c4]) = make_float4(ra[h * 4], ra[h * 4 + 1], ra[h * 4 + 2], ra[h * 4 + 3]);
            }
        }
    };
    auto store_b = [&](int buf) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int idx = tid + h * NT;
            if (TB) {
                const int r = idx >> 2, c4 = (idx & 3) * 4;
#pragma unroll
                for (int e = 0; e < 4; ++e) Bs[buf][c4 + e][r] = rb[h * 4 + e];
            } else {
                const int r = idx >> 5, c4 = (idx & 31) * 4;
                *reinterpret_cast<float4 *>(&Bs[buf][r][c4]) = make_float4(rb[h * 4], rb[h * 4 + 1], rb[h * 4 + 2], rb[h * 4 + 3]);
            }
        }
    };

    const int ntiles = (kend - kbeg + BK - 1) / BK;
    if (ntiles > 0) {
        load_a(kbeg);
        load_b(kbeg);
        store_a(0);
        store_b(0);
    }
    __syncthreads();
    for (int it = 0; it < ntiles; ++it) {
        const int buf = it & 1;
        if (it + 1 < ntiles) {
            load_a(kbeg + (it + 1) * BK);
            load_b(kbeg + (it + 1) * BK);
        }
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4 *>(&Bs[buf][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4 *>(&Bs[buf][k][64 + tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (it + 1 < ntiles) {
            store_a(buf ^ 1);
            store_b(buf ^ 1);
        }
        __syncthreads();
    }

    if (g.vecc) {       // 16 consecutive lanes store 16 consecutive float4 of a row: full 128-byte lines
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = m0 + ((i < 4) ? ty * 4 + i : 64 + ty * 4 + (i - 4));
            if (m >= g.M) continue;
#pragma unroll
            for (int jh = 0; jh < 2; ++jh) {
                const int n = n0 + jh * 64 + tx * 4;
                const float4 a4 = make_float4(acc[i][jh * 4], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]);
                if (n + 3 < g.N) {
                    if (g.partial) *reinterpret_cast<float4 *>(g.partial + ((int64_t)blockIdx.z * g.M + m) * g.N + n) = a4;
                    else *reinterpret_cast<float4 *>(g.C + (int64_t)m * g.ldc + n) = epilogue4(g, a4, m, n);
                } else {
                    const float av[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        if (n + e >= g.N) continue;
                        if (g.partial) g.partial[((int64_t)blockIdx.z * g.M + m) * g.N + n + e] = av[e];
                        else g.C[(int64_t)m * g.ldc + n + e] = epilogue(g, av[e], m, n + e);
                    }
                }
            }
        }
        return;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + ((i < 4) ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (m >= g.M) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = n0 + ((j < 4) ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            if (n >= g.N) continue;
            if (g.partial) g.partial[((int64_t)blockIdx.z * g.M + m) * g.N + n] = acc[i][j];
            else g.C[(int64_t)m * g.ldc + n] = epilogue(g, acc[i][j], m, n);
        }
    }
}

__global__ void splitk_reduce_kernel(GemmArgs g, int splits) {
    const int64_t total = (int64_t)g.M * g.N;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int z = 0; z < splits; ++z) s += g.partial[(int64_t)z * total + idx];
        const int m = (int)(idx / g.N), n = (int)(idx % g.N);
        g.C[(int64_t)m * g.ldc + n] = epilogue(g, s, m, n);
    }
}

static int choose_splits(int M, int N, int K) {
    const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
    const int sms = num_sms();
    if (tiles >= sms || K < 4 * BK * 8) return 1;
    int splits = (2 * sms + tiles - 1) / tiles;
    const int maxs = K / (BK * 8);   // at least 8 k-tiles per split
    if (splits > maxs) splits = maxs;
    if (splits > 64) splits = 64;
    return splits < 1 ? 1 : splits;
}

// The one place that decides how an FFMA contraction runs: ctcb_gemm_f32 and ctcb_debug_gemm_plan both call it.
// Splits need room for their partials in the ws_bytes of workspace; without it the contraction runs unsplit.
void gemm_simt_plan(int M, int N, int K, const float *A, int64_t lda, const float *B, int64_t ldb, size_t ws_bytes,
                    GemmSimtPlan *p) {
    int splits = choose_splits(M, N, K);
    if (splits > 1 && ws_bytes < (size_t)splits * M * N * sizeof(float)) splits = 1;
    int kps = (K + splits - 1) / splits;
    kps = (kps + BK - 1) / BK * BK;
    p->k_per_split = kps > 0 ? kps : BK;
    splits = K > 0 ? (K + p->k_per_split - 1) / p->k_per_split : 1;
    p->splits = splits > 1 ? splits : 1;
    p->vec = (lda % 4 == 0) && (ldb % 4 == 0) && (((uintptr_t)A | (uintptr_t)B) % 16 == 0);
    p->ctas = ((N + BN - 1) / BN) * ((M + BM - 1) / BM) * p->splits;
}

}  // namespace ctcb

namespace ctcb {
bool gemm_tc_eligible(int M, int N, int K);
size_t gemm_tc_workspace_bytes(int M, int N, int K);
int run_gemm_tc(int transA, int transB, int M, int N, int K, float alpha, const float *A, int64_t lda, const float *B,
                int64_t ldb, float beta, float *C, int64_t ldc, const float *bias, int relu, const float *mask_src,
                void *ws, size_t ws_bytes, cudaStream_t st);
size_t gemm_tc_pair_workspace_bytes(int M, int N, int K);
int run_gemm_tc_pair(int transA, int transB, int M, int N, int K, float alpha, const float *const *A, int64_t lda,
                     const float *const *B, int64_t ldb, float beta, float *const *C, int64_t ldc, void *ws,
                     size_t ws_bytes, cudaStream_t st);
}

using namespace ctcb;

extern "C" size_t ctcb_gemm_workspace_bytes(int M, int N, int K) {
    const int s = choose_splits(M, N, K);
    size_t simt = s > 1 ? (size_t)s * M * N * sizeof(float) : 0;
    size_t tc = gemm_tc_eligible(M, N, K) ? gemm_tc_workspace_bytes(M, N, K) : 0;
    return simt > tc ? simt : tc;
}

extern "C" int ctcb_gemm_f32(int transA, int transB, int M, int N, int K, float alpha, const float *A, int64_t lda,
                             const float *B, int64_t ldb, float beta, float *C, int64_t ldc, const float *bias,
                             int relu, const float *mask_src, void *workspace, size_t ws_bytes, void *stream) {
    if (M <= 0 || N <= 0) return CTCB_OK;
    if (!A || !B || !C || K < 0) return set_error(CTCB_EINVAL, "ctcb_gemm_f32: bad argument");
    if (M > GEMM_MAX_M) return set_error(CTCB_EINVAL, "ctcb_gemm_f32: M = %d exceeds %d rows", M, GEMM_MAX_M);
    // large contractions: 3xTF32 on the wgmma tensor cores (gemm_tc.cu); small or odd ones: exact FFMA below
    if (gemm_tc_eligible(M, N, K) && workspace && ws_bytes >= gemm_tc_workspace_bytes(M, N, K))
        return run_gemm_tc(transA, transB, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, bias, relu, mask_src, workspace,
                           ws_bytes, (cudaStream_t)stream);
    GemmArgs g;
    g.M = M; g.N = N; g.K = K; g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.C = C; g.ldc = ldc;
    g.alpha = alpha; g.beta = beta; g.bias = bias; g.relu = relu; g.mask = mask_src;
    GemmSimtPlan p;
    gemm_simt_plan(M, N, K, A, lda, B, ldb, workspace ? ws_bytes : 0, &p);
    const int splits = p.splits;
    const bool vec = p.vec;
    g.k_per_split = p.k_per_split;
    g.partial = splits > 1 ? (float *)workspace : nullptr;
    g.vecc = g.partial ? (N % 4 == 0 && ((uintptr_t)g.partial) % 16 == 0)
                       : (ldc % 4 == 0 && ((uintptr_t)C) % 16 == 0 && (!mask_src || ((uintptr_t)mask_src) % 16 == 0));
    dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, splits);
    cudaStream_t st = (cudaStream_t)stream;
#define GO(TA, TB)                                                                  \
    do {                                                                            \
        if (vec) gemm_simt_kernel<TA, TB, true><<<grid, NT, 0, st>>>(g);            \
        else gemm_simt_kernel<TA, TB, false><<<grid, NT, 0, st>>>(g);               \
    } while (0)
    if (!transA && !transB) GO(false, false);
    else if (!transA && transB) GO(false, true);
    else if (transA && !transB) GO(true, false);
    else GO(true, true);
#undef GO
    CTCB_LAUNCH_CHECK();
    if (splits > 1) {
        const int64_t total = (int64_t)M * N;
        int blocks = (int)((total + 255) / 256);
        if (blocks > 4 * num_sms()) blocks = 4 * num_sms();
        splitk_reduce_kernel<<<blocks, 256, 0, st>>>(g, splits);
        CTCB_LAUNCH_CHECK();
    }
    return CTCB_OK;
}

extern "C" size_t ctcb_gemm_pair_workspace_bytes(int M, int N, int K) {
    const size_t one = ctcb_gemm_workspace_bytes(M, N, K);
    const size_t tc = gemm_tc_eligible(M, N, K) ? gemm_tc_pair_workspace_bytes(M, N, K) : 0;
    return one > tc ? one : tc;
}

extern "C" int ctcb_gemm_pair_f32(int transA, int transB, int M, int N, int K, float alpha, const float *A0,
                                  const float *A1, int64_t lda, const float *B0, const float *B1, int64_t ldb,
                                  float beta, float *C0, float *C1, int64_t ldc, void *workspace, size_t ws_bytes,
                                  void *stream) {
    if (M <= 0 || N <= 0) return CTCB_OK;
    if (!A0 || !A1 || !B0 || !B1 || !C0 || !C1 || K < 0) return set_error(CTCB_EINVAL, "ctcb_gemm_pair_f32: bad argument");
    if (M > GEMM_MAX_M) return set_error(CTCB_EINVAL, "ctcb_gemm_pair_f32: M = %d exceeds %d rows", M, GEMM_MAX_M);
    if (gemm_tc_eligible(M, N, K) && workspace && ws_bytes >= gemm_tc_pair_workspace_bytes(M, N, K)) {
        const float *A[2] = {A0, A1}, *B[2] = {B0, B1};
        float *C[2] = {C0, C1};
        return run_gemm_tc_pair(transA, transB, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, workspace, ws_bytes,
                                (cudaStream_t)stream);
    }
    const int rc = ctcb_gemm_f32(transA, transB, M, N, K, alpha, A0, lda, B0, ldb, beta, C0, ldc, nullptr, 0, nullptr,
                                 workspace, ws_bytes, stream);
    if (rc != CTCB_OK) return rc;
    return ctcb_gemm_f32(transA, transB, M, N, K, alpha, A1, lda, B1, ldb, beta, C1, ldc, nullptr, 0, nullptr,
                         workspace, ws_bytes, stream);
}

// TF32 mode (include/ctcb200.h): the same calls with the planners in TF32 mode
extern "C" int ctcb_gemm_tf32(int transA, int transB, int M, int N, int K, float alpha, const float *A, int64_t lda,
                              const float *B, int64_t ldb, float beta, float *C, int64_t ldc, const float *bias,
                              int relu, const float *mask_src, void *workspace, size_t ws_bytes, void *stream) {
    Tf32Scope tf32(1);
    return ctcb_gemm_f32(transA, transB, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, bias, relu, mask_src, workspace,
                         ws_bytes, stream);
}
extern "C" int ctcb_gemm_pair_tf32(int transA, int transB, int M, int N, int K, float alpha, const float *A0,
                                   const float *A1, int64_t lda, const float *B0, const float *B1, int64_t ldb,
                                   float beta, float *C0, float *C1, int64_t ldc, void *workspace, size_t ws_bytes,
                                   void *stream) {
    Tf32Scope tf32(1);
    return ctcb_gemm_pair_f32(transA, transB, M, N, K, alpha, A0, A1, lda, B0, B1, ldb, beta, C0, C1, ldc, workspace,
                              ws_bytes, stream);
}
