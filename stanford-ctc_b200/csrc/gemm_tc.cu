// gemm_tc.cu -- fp32-faithful dense contraction on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// The reference multiplies in float32 (cudamat cm.dot -> legacy cuBLAS sgemm; call sites
// ctc_fast/nnets/brnnet.py:140,196,204,227-230).  The tensor cores have no fp32 MMA, and a single TF32 pass
// (10-bit mantissa) would be a reduced-precision run, so every operand is split into two TF32 parts
//     x = hi + lo,   hi = x with the low 13 mantissa bits cleared (what a .tf32 MMA reads from an fp32 word),
//                    lo = x - hi (exact in fp32; itself read as TF32)
// and a product is three MMAs accumulated in fp32:  lo.hi + hi.lo + hi.hi
// (the dropped lo.lo term is ~2^-20 relative) -- "3xTF32", ~1e-6 relative error per product.
//
// Kernel shape: C[M x N] = A[M x K] . B[N x K]^T, both operands K-major (wgmma reads .tf32 operands K-major only; an
// operand stored the other way round is transposed by a prep kernel first).  One CTA (3 warpgroups) per 128 x BN output
// tile and K split (gridDim.z):
//   warpgroup 0 : producer -- one elected thread TMA-loads the A and B tiles of each k-block of 32 floats into a
//                 STAGES-deep ring (mbarrier complete_tx); the 128 threads then write the low halves of both tiles
//                 next to them (element-wise, oblivious to the swizzle) and signal the consumers;
//   warpgroups 1, 2 : consumers -- rows 0..63 / 64..127 of the tile: 4 k-steps x 3 wgmma (m64 x BN x k8) per k-block
//                 with the accumulator in registers, one k-block in flight while the previous slot is released; then
//                 the fused alpha/beta/bias/ReLU/mask epilogue (or the split-K partial) straight from registers.
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <stdlib.h>

namespace ctcb {

constexpr int TC_BM = 128;
constexpr int TC_BK = 32;   // 32 fp32 = 128 bytes = one swizzle span
constexpr int TC_THREADS = 384;

static unsigned long long *g_gemm_trace = nullptr;     // CTCB_GEMM_TRACE: stamps of the LAST tensor-core GEMM launched

struct GemmTcArgs {
    int M, N, K;
    float *C; int64_t ldc;
    float alpha, beta;
    const float *bias; int relu; const float *mask;
    float *partial;      // split-K partials [splits][M][N] or nullptr
    int kb_per_split;    // k-blocks per gridDim.z slice
    unsigned long long *trace;   // optional (CTCB_GEMM_TRACE): [64 k-blocks][8] SM clock stamps of CTA (0,0,0)
};
#define TC_STAMP(i, slot)                                                                                       \
    do {                                                                                                        \
        if (g.trace && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && (i) < 64)                       \
            g.trace[(i) * 8 + (slot)] = (unsigned long long)clock64();                                          \
    } while (0)

// ---------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t tc_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tc_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void tc_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tc_mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool tc_mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait: a protocol bug becomes a trap (CUDA error), never a hung GPU
__device__ __forceinline__ void tc_mbar_wait(uint32_t bar, uint32_t parity) {
    if (tc_mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!tc_mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();
    }
}
__device__ __forceinline__ void tc_tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}

__device__ __forceinline__ float tc_epilogue(const GemmTcArgs &g, float acc, int m, int n) {
    float v = g.alpha * acc;
    if (g.beta != 0.f) v += g.beta * g.C[(int64_t)m * g.ldc + n];
    if (g.bias) v += g.bias[n];
    if (g.relu) v = fmaxf(v, 0.f);
    if (g.mask) v = (g.mask[(int64_t)m * g.ldc + n] > 0.f) ? v : 0.f;
    return v;
}

__device__ __forceinline__ float4 tc_lo4(float4 v) {
    float4 r;
    r.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xffffe000u);
    r.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xffffe000u);
    r.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xffffe000u);
    r.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xffffe000u);
    return r;
}

// A stage holds [A value | A low half | B value | B low half], each tile 1024-byte aligned.
template <int BN, int STAGES>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmTcArgs g) {
    constexpr uint32_t A_BYTES = TC_BM * TC_BK * 4, B_BYTES = BN * TC_BK * 4;
    constexpr uint32_t B_OFF = 2 * A_BYTES;
    constexpr uint32_t STAGE_BYTES = B_OFF + 2 * B_BYTES;
    extern __shared__ __align__(1024) uint8_t tc_smem[];
    // 1024-byte alignment is required by SWIZZLE_128B: align manually (dynamic smem base is only 16B-aligned by contract)
    uint8_t *base = (uint8_t *)(((uintptr_t)tc_smem + 1023) & ~(uintptr_t)1023);
    // full[STAGES] (TMA landed), empty[STAGES] (consumers done with the slot), ready[STAGES] (low halves written)
    uint64_t *full = reinterpret_cast<uint64_t *>(base + STAGES * STAGE_BYTES);
    uint64_t *empty = full + STAGES, *ready = full + 2 * STAGES;

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * TC_BM, n0 = blockIdx.x * BN;
    const int nkb_total = (g.K + TC_BK - 1) / TC_BK;
    const int kb0 = blockIdx.z * g.kb_per_split;
    const int kb1 = min(nkb_total, kb0 + g.kb_per_split);
    const int nkb = kb1 - kb0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            tc_mbar_init(tc_smem_u32(&full[s]), 1);
            tc_mbar_init(tc_smem_u32(&empty[s]), 8);    // one arrival per consumer warp
            tc_mbar_init(tc_smem_u32(&ready[s]), 4);    // one arrival per producer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        // ---------------------------------------------------------------- producer: TMA issue runs STAGES - 1 k-blocks
        // ahead of the split.  Split first, then issue: the slot of block i is freed by the consumers once they have
        // started on block i - STAGES + 1, whose low halves this very iteration provides.
        if (threadIdx.x == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
        }
        constexpr int LA = STAGES - 1;
        constexpr int NQ = (int)((A_BYTES + B_BYTES) / 16) / 128;
        for (int i = 0; i < nkb + LA; ++i) {
            const int j = i - LA;
            if (j >= 0) {
                const int s = j % STAGES, use = j / STAGES;
                tc_mbar_wait(tc_smem_u32(&full[s]), (uint32_t)(use & 1));
                if (threadIdx.x == 0) TC_STAMP(j, 1);
                uint8_t *st = base + s * STAGE_BYTES;
                float4 v[NQ];       // every load first, then every store
#pragma unroll
                for (int q = 0; q < NQ; ++q) {
                    const int idx = threadIdx.x + 128 * q;                  // float4 index over A then B
                    const int aq = (int)(A_BYTES / 16);
                    v[q] = idx < aq ? reinterpret_cast<const float4 *>(st)[idx]
                                    : reinterpret_cast<const float4 *>(st + B_OFF)[idx - aq];
                }
#pragma unroll
                for (int q = 0; q < NQ; ++q) {
                    const int idx = threadIdx.x + 128 * q;
                    const int aq = (int)(A_BYTES / 16);
                    if (idx < aq) reinterpret_cast<float4 *>(st + A_BYTES)[idx] = tc_lo4(v[q]);
                    else reinterpret_cast<float4 *>(st + B_OFF + B_BYTES)[idx - aq] = tc_lo4(v[q]);
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic writes -> tensor-core (async) proxy
                __syncwarp();
                if (lane == 0) tc_mbar_arrive(tc_smem_u32(&ready[s]));
                if (threadIdx.x == 0) TC_STAMP(j, 2);
            }
            if (i < nkb && threadIdx.x == 0) {
                const int s = i % STAGES, use = i / STAGES;
                if (use > 0) tc_mbar_wait(tc_smem_u32(&empty[s]), (uint32_t)((use - 1) & 1));
                const uint32_t fb = tc_smem_u32(&full[s]);
                const uint32_t sa = tc_smem_u32(base + s * STAGE_BYTES);
                const int k = (kb0 + i) * TC_BK;
                TC_STAMP(i, 0);
                tc_mbar_expect_tx(fb, A_BYTES + B_BYTES);
                tc_tma_load_2d(sa, &tmA, fb, k, m0);
                tc_tma_load_2d(sa + B_OFF, &tmB, fb, k, n0);
            }
        }
        return;
    }

    // -------------------------------------------------------------------- consumers
    const int cw = wg - 1;                                        // rows 64 cw .. 64 cw + 63 of the tile
    float acc[BN / 2];
#pragma unroll
    for (int r = 0; r < BN / 2; ++r) acc[r] = 0.f;
    for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES, use = i / STAGES;
        tc_mbar_wait(tc_smem_u32(&ready[s]), (uint32_t)(use & 1));      // hi landed and lo written
        if (threadIdx.x == 128) TC_STAMP(i, 3);
        const uint32_t sa = tc_smem_u32(base + s * STAGE_BYTES) + (uint32_t)cw * (64 * 128);
        const uint32_t sb = tc_smem_u32(base + s * STAGE_BYTES) + B_OFF;
        const uint64_t dA = wg_desc(sa), dAl = wg_desc(sa + A_BYTES), dB = wg_desc(sb), dBl = wg_desc(sb + B_BYTES);
        wg_fence();
#pragma unroll
        for (int k8 = 0; k8 < TC_BK / 8; ++k8) {
            const uint64_t adv = (uint64_t)((k8 * 32) >> 4);
            WgmmaTf32<BN>::mma(acc, dAl + adv, dB + adv, (i > 0 || k8 > 0) ? 1u : 0u);   // lo . hi
            WgmmaTf32<BN>::mma(acc, dA + adv, dBl + adv, 1u);                            // hi . lo
            WgmmaTf32<BN>::mma(acc, dA + adv, dB + adv, 1u);                             // hi . hi
        }
        wg_commit();
        if (threadIdx.x == 128) TC_STAMP(i, 4);
        // the previous k-block's MMAs are complete once at most this one is outstanding: release its slot
        wg_wait<1>();
        if (i > 0) {
            __syncwarp();
            if (lane == 0) tc_mbar_arrive(tc_smem_u32(&empty[(i - 1) % STAGES]));
        }
    }
    wg_wait<0>();
    // (the last slot is never waited for again: nothing is loaded after it)

    // -------------------------------------------------------------------- epilogue straight from the accumulator
    const int q = warp & 3;
    const int rbase = m0 + 64 * cw + 16 * q + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = rbase + 8 * h;
        if (m >= g.M) continue;
        float *drow = g.partial ? g.partial + ((int64_t)blockIdx.z * g.M + m) * g.N : g.C + (int64_t)m * g.ldc;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int n = n0 + 8 * j + 2 * (lane & 3);
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if (!g.partial) {
                if (n < g.N) v0 = tc_epilogue(g, v0, m, n);
                if (n + 1 < g.N) v1 = tc_epilogue(g, v1, m, n + 1);
            }
            if (n + 1 < g.N && (((uintptr_t)(drow + n)) & 7) == 0) {
                *reinterpret_cast<float2 *>(drow + n) = make_float2(v0, v1);
            } else {
                if (n < g.N) drow[n] = v0;
                if (n + 1 < g.N) drow[n + 1] = v1;
            }
        }
    }
}

// ---------------------------------------------------------------------------------- prep kernels
// out_lo[r][c] = x - trunc_tf32(x); optionally out_hi = x re-pitched.  No transpose: rows x cols, ld -> ldo.
__global__ void tc_split_kernel(const float *__restrict__ x, int64_t ld, int rows, int cols, float *__restrict__ hi,
                                float *__restrict__ lo, int64_t ldo) {
    const int64_t total = (int64_t)rows * ldo;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(idx / ldo), c = (int)(idx - (int64_t)r * ldo);
        const float v = (c < cols) ? x[(int64_t)r * ld + c] : 0.f;
        const float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
        if (hi) hi[idx] = v;
        if (lo) lo[idx] = v - h;
    }
}
// transposing variant: x is rows x cols (ld); outputs are cols x rows (ldo >= rows), tiled through shared memory
__global__ void tc_split_transpose_kernel(const float *__restrict__ x, int64_t ld, int rows, int cols,
                                          float *__restrict__ hi, float *__restrict__ lo, int64_t ldo) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < rows && c < cols) ? x[(int64_t)r * ld + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + threadIdx.x;     // output row = c, output col = r
        if (c < cols && r < ldo) {
            const float v = (r < rows) ? tile[threadIdx.x][i] : 0.f;
            const float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
            hi[(int64_t)c * ldo + r] = v;
            if (lo) lo[(int64_t)c * ldo + r] = v - h;
        }
    }
}

__global__ void tc_splitk_reduce_kernel(GemmTcArgs g, int splits) {
    const int64_t total = (int64_t)g.M * g.N;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int z = 0; z < splits; ++z) s += g.partial[(int64_t)z * total + idx];
        const int m = (int)(idx / g.N), n = (int)(idx % g.N);
        g.C[(int64_t)m * g.ldc + n] = tc_epilogue(g, s, m, n);
    }
}

// ---------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
        else
            cudaGetLastError();
    }
    return fn;
}

// rows x K fp32, K-major with pitch ld (elements); box = 32 floats x box_rows, 128B swizzle, OOB -> 0
static int make_map(CUtensorMap *m, const float *ptr, int rows, int K, int64_t ld, int box_rows) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return set_error(CTCB_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(CTCB_ECUDA, "cuTensorMapEncodeTiled failed (%d) rows=%d K=%d ld=%lld", (int)r, rows, K, (long long)ld);
    return CTCB_OK;
}

static inline int64_t pad4(int64_t x) { return (x + 3) / 4 * 4; }

// 64-wide tiles for narrow outputs (the accumulator then takes 32 registers per thread instead of 64)
static int tc_pick_bn(int N) { return N <= 64 ? 64 : 128; }

// The tensor cores' fp32 accumulation does not round to nearest, so the relative error of one accumulator chain grows
// linearly with its length (tools/gemm_check.py big shows it).  No chain is allowed to be longer than TC_CHAIN_KB
// k-blocks (K = 2048): longer contractions are split over K and the partial sums are added in fp32 with
// round-to-nearest by the reduce kernel (deterministic order).
constexpr int TC_CHAIN_KB = 64;

static int tc_choose_splits(int M, int N, int K, int BN) {
    const int tiles = ((M + TC_BM - 1) / TC_BM) * ((N + BN - 1) / BN);
    const int nkb = (K + TC_BK - 1) / TC_BK;
    const int sms = num_sms();
    int splits = 1;
    if (tiles < sms && nkb >= 16) {          // fill the device
        splits = (sms + tiles - 1) / tiles;
        if (splits > nkb / 8) splits = nkb / 8;
        if (splits > 32) splits = 32;
        if (splits < 1) splits = 1;
    }
    const int need = (nkb + TC_CHAIN_KB - 1) / TC_CHAIN_KB;     // bound the accumulator chain
    if (splits < need) splits = need;
    return splits;
}

bool gemm_tc_enabled() {
    static int on = -1;
    if (on < 0) {
        const char *e = getenv("CTCB_GEMM");
        on = (e && e[0] == 's') ? 0 : 1;     // CTCB_GEMM=simt forces the FFMA kernel everywhere
        if (on && !get_encode()) on = 0;
    }
    return on == 1;
}

// Below these sizes the exact FFMA kernel is used: short contractions (K = 41 / 62) would need re-pitched copies and
// cannot amortise the tensor-core pipeline.  The thresholds have not been re-tuned on H100.
bool gemm_tc_eligible(int M, int N, int K) {
    static int min_k = -1, min_m = -1;      // CTCB_GEMM_MINK / _MINM: smallest contraction length / row count that goes to the tensor cores
    if (min_k < 0) { const char *e = getenv("CTCB_GEMM_MINK"); min_k = e ? atoi(e) : 128; }
    if (min_m < 0) { const char *e = getenv("CTCB_GEMM_MINM"); min_m = e ? atoi(e) : 32; }
    return gemm_tc_enabled() && M >= min_m && N >= 32 && K >= min_k;
}

size_t gemm_tc_workspace_bytes(int M, int N, int K) {
    const int64_t Kp = pad4(K);
    size_t prep = ((size_t)M * Kp + (size_t)N * Kp) * sizeof(float);     // re-laid-out copies of A and B (when needed)
    const int BN = tc_pick_bn(N);
    const int splits = tc_choose_splits(M, N, K, BN);
    size_t part = splits > 1 ? (size_t)splits * M * N * sizeof(float) : 0;
    return align_up(prep, 256) + align_up(part, 256) + 1024;
}

template <int BN, int STAGES>
static int launch_tc(const CUtensorMap &tA, const CUtensorMap &tB, const GemmTcArgs &g, int splits, cudaStream_t st) {
    constexpr size_t smem = (size_t)STAGES * (2 * TC_BM * TC_BK * 4 + 2 * BN * TC_BK * 4) + 3 * STAGES * 8 + 1024;
    static_assert(smem <= 227 * 1024, "stage ring exceeds the shared memory of a block");
    CTCB_CUDA_CHECK(cudaFuncSetAttribute((gemm_tc_kernel<BN, STAGES>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((g.N + BN - 1) / BN, (g.M + TC_BM - 1) / TC_BM, splits);
    gemm_tc_kernel<BN, STAGES><<<grid, TC_THREADS, smem, st>>>(tA, tB, g);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

// Same contract as ctcb_gemm_f32; ws must hold gemm_tc_workspace_bytes(M, N, K).
int run_gemm_tc(int transA, int transB, int M, int N, int K, float alpha, const float *A, int64_t lda, const float *B,
                int64_t ldb, float beta, float *C, int64_t ldc, const float *bias, int relu, const float *mask_src,
                void *ws, size_t ws_bytes, cudaStream_t st) {
    if (ws_bytes < gemm_tc_workspace_bytes(M, N, K)) return set_error(CTCB_ENOMEM, "run_gemm_tc: workspace too small");
    const int64_t Kp = pad4(K);
    float *p = (float *)ws;
    float *Ahi = p; p += (size_t)M * Kp;
    float *Bhi = p; p += (size_t)N * Kp;
    float *part = (float *)((char *)ws + align_up(((size_t)M * Kp + (size_t)N * Kp) * sizeof(float), 256));

    // ---- operand A as M x K, K-major: stored M x K (transA=0) or K x M (transA=1, transposed into a copy)
    const float *Ause; int64_t lda_use;
    auto ew_grid = [](int64_t n) { int64_t b = (n + 255) / 256; const int cap = 16 * num_sms(); return (int)(b > cap ? cap : (b < 1 ? 1 : b)); };
    if (transA) {
        tc_split_transpose_kernel<<<dim3((M + 31) / 32, (K + 31) / 32), dim3(32, 8), 0, st>>>(A, lda, K, M, Ahi, nullptr, Kp);
        CTCB_LAUNCH_CHECK();
        Ause = Ahi; lda_use = Kp;
    } else if ((lda % 4 == 0) && (((uintptr_t)A) % 16 == 0)) {
        Ause = A; lda_use = lda;                       // TMA reads the caller's array directly
    } else {
        tc_split_kernel<<<ew_grid((int64_t)M * Kp), 256, 0, st>>>(A, lda, M, K, Ahi, nullptr, Kp);   // re-pitch to 16-byte rows
        CTCB_LAUNCH_CHECK();
        Ause = Ahi; lda_use = Kp;
    }
    // ---- operand B as N x K, K-major: stored N x K (transB=1) or K x N (transB=0, transposed into a copy)
    const float *Buse; int64_t ldb_use;
    if (!transB) {
        tc_split_transpose_kernel<<<dim3((N + 31) / 32, (K + 31) / 32), dim3(32, 8), 0, st>>>(B, ldb, K, N, Bhi, nullptr, Kp);
        CTCB_LAUNCH_CHECK();
        Buse = Bhi; ldb_use = Kp;
    } else if ((ldb % 4 == 0) && (((uintptr_t)B) % 16 == 0)) {
        Buse = B; ldb_use = ldb;
    } else {
        tc_split_kernel<<<ew_grid((int64_t)N * Kp), 256, 0, st>>>(B, ldb, N, K, Bhi, nullptr, Kp);
        CTCB_LAUNCH_CHECK();
        Buse = Bhi; ldb_use = Kp;
    }

    const int BN = tc_pick_bn(N);
    int splits = tc_choose_splits(M, N, K, BN);
    const int nkb = (K + TC_BK - 1) / TC_BK;
    GemmTcArgs g;
    g.M = M; g.N = N; g.K = K; g.C = C; g.ldc = ldc; g.alpha = alpha; g.beta = beta; g.bias = bias; g.relu = relu; g.mask = mask_src;
    g.trace = nullptr;
    {
        static int tr_env = -1;
        if (tr_env < 0) tr_env = getenv("CTCB_GEMM_TRACE") ? 1 : 0;
        if (tr_env) {
            if (!g_gemm_trace) cudaMalloc(&g_gemm_trace, 64 * 8 * sizeof(unsigned long long));
            g.trace = g_gemm_trace;
        }
    }
    g.kb_per_split = (nkb + splits - 1) / splits;
    splits = (nkb + g.kb_per_split - 1) / g.kb_per_split;
    g.partial = splits > 1 ? part : nullptr;

    CUtensorMap tA, tB;
    int rc;
    if ((rc = make_map(&tA, Ause, M, K, lda_use, TC_BM)) != CTCB_OK) return rc;
    if ((rc = make_map(&tB, Buse, N, K, ldb_use, BN)) != CTCB_OK) return rc;
    // 192 KB of ring either way: 4 stages of 48 KB (64-wide) or 3 of 64 KB (128-wide)
    rc = (BN == 64) ? launch_tc<64, 4>(tA, tB, g, splits, st) : launch_tc<128, 3>(tA, tB, g, splits, st);
    if (rc != CTCB_OK) return rc;
    if (splits > 1) {
        const int64_t total = (int64_t)M * N;
        int blocks = (int)((total + 255) / 256);
        if (blocks > 4 * num_sms()) blocks = 4 * num_sms();
        tc_splitk_reduce_kernel<<<blocks, 256, 0, st>>>(g, splits);
        CTCB_LAUNCH_CHECK();
    }
    return CTCB_OK;
}

}  // namespace ctcb

// Diagnostic: the per-k-block clock stamps of CTA (0,0,0) of the last tensor-core GEMM (CTCB_GEMM_TRACE=1):
// [64][8] = {TMA issued, tile landed, lo written, consumers saw it, MMAs issued}.  Returns 0 when tracing is off.
extern "C" int ctcb_debug_gemm_trace(unsigned long long *host_out) {
    if (!ctcb::g_gemm_trace || !host_out) return 0;
    if (cudaMemcpy(host_out, ctcb::g_gemm_trace, 64 * 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
    return 64;
}
