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
// Kernel shape: C[M x N] = A[M x K] . B[N x K]^T.  wgmma reads .tf32 operands K-major only.  A reaches the MMAs from
// registers, B from shared memory by descriptor, 128-byte swizzled:
//   A: TMA writes the tile 128B-swizzled into the A slot, as one [rows][32 k] box (K-major, [M][K]) or as four
//     [32 k][32 rows] boxes (MN-major, [K][M], e.g. the time-major deltas of a weight gradient over T*B rows); each
//     consumer loads its fragments from it and splits them into hi and lo in registers (tc_load_split_a), conflict-free.
//   B: a K-major tile ([N][K]) lands swizzled in the value slot; an MN-major one ([K][N]) lands unswizzled in the
//     LOW-HALF slot and the producer transposes it into the swizzled value slot while it computes the low halves.  The
//     wgmma then reads the same bytes as if a transposed copy had been loaded, so both ways give identical results.
//   An operand TMA cannot describe (row pitch not a multiple of 16 bytes, base not 16-byte aligned) is re-pitched or
//   transposed into the workspace by a prep kernel first (also forced by CTCB_GEMM_TC_COPY=1).
// One CTA (3 warpgroups) per 128 x BN output tile, K split and problem (gridDim.z = problems x splits):
//   warpgroup 0 : producer -- one elected thread TMA-loads the A and B tiles of each k-block of 32 floats into a
//                 STAGES-deep ring (mbarrier complete_tx); the 128 threads then write the low half of the B tile next
//                 to it (and its transposed values when it is MN-major) and signal the consumers;
//   warpgroups 1, 2 : consumers -- rows 0..63 / 64..127 of the tile: per k-block, load and split the A fragments, then
//                 4 k-steps x 3 wgmma (m64 x BN x k8, A from registers) with the accumulator in registers, wait for them
//                 and release the slot; then the fused alpha/beta/bias/ReLU/mask epilogue (or the split-K partial)
//                 straight from registers.
// Each product sees the same hi and lo values and the MMAs run in the same order whichever way an operand arrives, so
// the results do not depend on the operand path.
// Two problems of the same shape (the two recurrent weight gradients) can share one launch and one split-K reduce.
//
// TF32 mode (include/ctcb200.h; gemm_tc_tf32_kernel, planned while a Tf32Scope is on): each operand is rounded to the
// nearest TF32 value (cvt.rna) instead of split, and a product is ONE MMA.  The consumers round their A fragments in
// registers; the producer rewrites B's value slot rounded (in place when K-major, in the transpose when MN-major), so
// no low half is written and a K-major B needs no second slot: the ring takes as many of these smaller stages as fit
// in the fp32-faithful ring's shared memory (tc_tf32_stages).  Copied operands stay exact in the workspace and are
// rounded in the ring like the others (rounding is idempotent).  BN, the K splits, the operand paths, the pair
// decision and the workspace are the fp32-faithful plan's.  With a third of the MMAs a k-block is no longer bound by
// the tensor pipe: on an H100 the traced k-block period falls from about 1920 to 1270 SM clocks (K-major 48000 x
// 2048 x 2048), of which the MMA issue is about 375; the rest is the operand stream (32 KB per CTA per k-block, about
// 6.6 TB/s from L2 over the 132 SMs), DESIGN.md section 6.
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
    float *C[2]; int64_t ldc;    // output of problem 0 / 1 (a second problem has no bias, ReLU or mask)
    float alpha, beta;
    const float *bias; int relu; const float *mask;
    float *partial;      // split-K partials [problems][splits][M][N] (row blockIdx.z) or nullptr
    int kb_per_split;    // k-blocks per split
    int splits;          // K splits per problem: blockIdx.z = problem * splits + split
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

__device__ __forceinline__ float tc_epilogue(const GemmTcArgs &g, const float *C, float acc, int m, int n) {
    float v = g.alpha * acc;
    if (g.beta != 0.f) v += g.beta * C[(int64_t)m * g.ldc + n];
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

// The producer's share of one ROWS x 32 operand tile: ROWS * 32 / 4 / 128 float4 per thread.
//   K-major (MN = false): the tile landed swizzled in `hi`; thread t takes float4 t, t + 128, ... in storage order and
//     writes their low halves to the same places in `lo` (the swizzle does not matter element-wise).
//   MN-major (MN = true): the tile landed in `lo` as [32 k][ROWS]; thread t takes row r = t % ROWS and the k-quads
//     c = t / ROWS + (128 / ROWS) q.  Reads: a warp reads 32 consecutive rows of one k, conflict-free.  Writes: element
//     (r, k) of a K-major 128B-swizzled tile lies at r * 128 + ((k / 4) ^ (r % 8)) * 16 + (k % 4) * 4, so each of the 8
//     threads of a 16-byte store phase (8 consecutive r, one c) hits a different 16-byte bank group: conflict-free.
//     Every thread must have loaded before any thread stores, since the stores overwrite `lo`.
template <int ROWS, bool MN>
struct TcTile {
    static constexpr int Q = ROWS * TC_BK / 4 / 128;
    static __device__ __forceinline__ void load(const uint8_t *hi, const uint8_t *lo, float4 (&v)[Q]) {
        if (MN) {
            const float *src = reinterpret_cast<const float *>(lo);
            const int r = threadIdx.x % ROWS, c0 = threadIdx.x / ROWS;
#pragma unroll
            for (int q = 0; q < Q; ++q) {
                const int k = 4 * (c0 + (128 / ROWS) * q);
                v[q] = make_float4(src[k * ROWS + r], src[(k + 1) * ROWS + r], src[(k + 2) * ROWS + r], src[(k + 3) * ROWS + r]);
            }
        } else {
#pragma unroll
            for (int q = 0; q < Q; ++q) v[q] = reinterpret_cast<const float4 *>(hi)[threadIdx.x + 128 * q];
        }
    }
    static __device__ __forceinline__ void store(uint8_t *hi, uint8_t *lo, const float4 (&v)[Q]) {
        if (MN) {
            const int r = threadIdx.x % ROWS, c0 = threadIdx.x / ROWS;
#pragma unroll
            for (int q = 0; q < Q; ++q) {
                const int off = r * 128 + (((c0 + (128 / ROWS) * q) ^ (r & 7)) << 4);
                *reinterpret_cast<float4 *>(hi + off) = v[q];
                *reinterpret_cast<float4 *>(lo + off) = tc_lo4(v[q]);
            }
        } else {
#pragma unroll
            for (int q = 0; q < Q; ++q) reinterpret_cast<float4 *>(lo)[threadIdx.x + 128 * q] = tc_lo4(v[q]);
        }
    }
    // TF32 mode: the value slot `hi` receives the values rounded to TF32 (in place when K-major), and `lo` only serves
    // as the MN-major landing area.
    static __device__ __forceinline__ void store_rna(uint8_t *hi, const float4 (&v)[Q]) {
        if (MN) {
            const int r = threadIdx.x % ROWS, c0 = threadIdx.x / ROWS;
#pragma unroll
            for (int q = 0; q < Q; ++q)
                *reinterpret_cast<float4 *>(hi + r * 128 + (((c0 + (128 / ROWS) * q) ^ (r & 7)) << 4)) = tf32_rna4(v[q]);
        } else {
#pragma unroll
            for (int q = 0; q < Q; ++q) reinterpret_cast<float4 *>(hi)[threadIdx.x + 128 * q] = tf32_rna4(v[q]);
        }
    }
};

// The consumers' A fragments (WgmmaTf32Rs) of one k-block, read from the A slot and split in registers: hi[4 kk + i] is
// register i of k-step kk as stored (the MMA reads its TF32 part), lo the same minus its TF32 part, tc_lo4's arithmetic.
// Thread (warp q of consumer cw, lane = 4 g + t) holds the tile rows of fragment rows g and g + 8 at k = 8 kk + t (+ 4).
//   K-major A (one 128 x 32 box, 128B-swizzled): row r at r * 128, k-quad c at ((c ^ (r % 8)) << 4), with fragment row
//     r = 64 cw + 16 q + g (+ 8), so r % 8 = g.  A warp's load reads k-quad 2 kk (+ 1) ^ g for its 8 g and word t of
//     it: 32 different banks.
//   MN-major A (four 32 k x 32 m boxes, 128B-swizzled, box j holds rows 32 j .. 32 j + 31): element (m, k) of a box lies
//     at k * 128 + (((m / 4) ^ (k % 8)) << 4) + (m % 4) * 4, so the bank is 4 ((m / 4) ^ (k % 8)) + m % 4.  Reading the
//     fragment rows as consecutive m (the warp reads 8 m x 4 k) would put two lanes on each bank.  So fragment row
//     (q, g, h) of consumer cw (h: the + 8 row) reads tile row  64 cw + 32 (q / 2) + 8 (q % 2) + 4 h + 16 (g / 4) + g % 4
//     (a bijection of the 128 rows; tc_tile_row gives it to the epilogue): the 8 g of a load take the m-quads
//     c and c + 4 (c = 2 (q % 2) + h) and m % 4 = g % 4, so with k % 8 = t (+ 4) the banks 4 ((c + 4 (g / 4)) ^ k % 8) + g % 4
//     are 32 different ones.
template <bool A_MN>
__device__ __forceinline__ int tc_tile_row(int cw, int q, int g, int h) {
    return A_MN ? 64 * cw + 32 * (q >> 1) + 8 * (q & 1) + 4 * h + 16 * (g >> 2) + (g & 3) : 64 * cw + 16 * q + g + 8 * h;
}
// TF32 = true: hi receives the values rounded to TF32 instead, and lo is not written.
template <bool A_MN, bool TF32>
__device__ __forceinline__ void tc_load_split_a(uint32_t sA, int cw, int q, int g, int t, uint32_t (&hi)[16],
                                                uint32_t (&lo)[16]) {
    // offsets of k-step kk, register i: the swizzle bits (4..6) are XORed in, the rest added
    const uint32_t p = A_MN ? sA + (2 * cw + (q >> 1)) * 4096 + t * 128 + (((2 * (q & 1) + 4 * (g >> 2)) ^ t) << 4) + (g & 3) * 4
                            : sA + (64 * cw + 16 * q + g) * 128 + (g << 4) + t * 4;
#pragma unroll
    for (int kk = 0; kk < TC_BK / 8; ++kk) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t a = A_MN ? ((p + kk * 1024 + (i >> 1) * 512) ^ (((i & 1) << 4) | ((i >> 1) << 6)))
                                    : ((p ^ ((2 * kk + (i >> 1)) << 4)) + (i & 1) * 1024);
            uint32_t x;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(x) : "r"(a));
            if (TF32) {
                hi[4 * kk + i] = tf32_rna(__uint_as_float(x));
            } else {
                hi[4 * kk + i] = x;
                lo[4 * kk + i] = __float_as_uint(__fsub_rn(__uint_as_float(x), __uint_as_float(x & 0xffffe000u)));
            }
        }
    }
}

// Bytes of one ring stage: [A value | B value | B low half], each tile 1024-byte aligned.  TF32 mode has no low half;
// the slot stays only as the landing area of an MN-major B.
template <int BN, bool B_MN, bool TF32>
__host__ __device__ constexpr uint32_t tc_stage_bytes() {
    return TC_BM * TC_BK * 4 + ((TF32 && !B_MN) ? 1 : 2) * BN * TC_BK * 4;
}

// A_MN / B_MN: the operand is MN-major in global memory (A: four swizzled 32-row boxes, see tc_load_split_a; B: its TMA
// box lands in the low-half slot, see TcTile).  TF32: one MMA of the operands rounded to TF32 per k8 step (the kernel
// gemm_tc_tf32_kernel), else three of their hi and lo parts (gemm_tc_kernel).
template <int BN, int STAGES, bool A_MN, bool B_MN, bool TF32>
__device__ __forceinline__ void gemm_tc_body(const CUtensorMap &tmA0, const CUtensorMap &tmB0, const CUtensorMap &tmA1,
                                             const CUtensorMap &tmB1, const GemmTcArgs &g) {
    constexpr uint32_t A_BYTES = TC_BM * TC_BK * 4, B_BYTES = BN * TC_BK * 4;
    constexpr uint32_t B_OFF = A_BYTES;
    constexpr uint32_t STAGE_BYTES = tc_stage_bytes<BN, B_MN, TF32>();
    extern __shared__ __align__(1024) uint8_t tc_smem[];
    // 1024-byte alignment is required by SWIZZLE_128B: align manually (dynamic smem base is only 16B-aligned by contract)
    uint8_t *base = (uint8_t *)(((uintptr_t)tc_smem + 1023) & ~(uintptr_t)1023);
    // full[STAGES] (TMA landed), empty[STAGES] (consumers done with the slot), ready[STAGES] (B's low half written)
    uint64_t *full = reinterpret_cast<uint64_t *>(base + STAGES * STAGE_BYTES);
    uint64_t *empty = full + STAGES, *ready = full + 2 * STAGES;

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * TC_BM, n0 = blockIdx.x * BN;
    const int prob = blockIdx.z / g.splits;
    const int nkb_total = (g.K + TC_BK - 1) / TC_BK;
    const int kb0 = (blockIdx.z - prob * g.splits) * g.kb_per_split;
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
        // finished block i - STAGES, and they can only start the block after it once this very iteration provides it.
        const CUtensorMap *tmA = prob ? &tmA1 : &tmA0, *tmB = prob ? &tmB1 : &tmB0;
        if (threadIdx.x == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(tmA) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(tmB) : "memory");
        }
        constexpr int LA = STAGES - 1;
        // an MN-major B box lands in the low-half slot, a K-major one in the value slot
        constexpr uint32_t B_DST = B_OFF + (B_MN ? B_BYTES : 0);
        for (int i = 0; i < nkb + LA; ++i) {
            const int j = i - LA;
            if (j >= 0) {
                const int s = j % STAGES, use = j / STAGES;
                tc_mbar_wait(tc_smem_u32(&full[s]), (uint32_t)(use & 1));
                if (threadIdx.x == 0) TC_STAMP(j, 1);
                uint8_t *st = base + s * STAGE_BYTES;
                float4 vb[TcTile<BN, B_MN>::Q];    // every load first, then every store
                TcTile<BN, B_MN>::load(st + B_OFF, st + B_OFF + B_BYTES, vb);
                if (B_MN) asm volatile("bar.sync 1, 128;" ::: "memory");   // the producer warpgroup only
                if (TF32)
                    TcTile<BN, B_MN>::store_rna(st + B_OFF, vb);
                else
                    TcTile<BN, B_MN>::store(st + B_OFF, st + B_OFF + B_BYTES, vb);
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
                // coordinates innermost first: (k, row) for a K-major map, (row, k) for an MN-major one
                if (A_MN) {
#pragma unroll
                    for (int b = 0; b < TC_BM / 32; ++b) tc_tma_load_2d(sa + b * 4096, tmA, fb, m0 + 32 * b, k);
                } else {
                    tc_tma_load_2d(sa, tmA, fb, k, m0);
                }
                tc_tma_load_2d(sa + B_DST, tmB, fb, B_MN ? n0 : k, B_MN ? k : n0);
            }
        }
        return;
    }

    // -------------------------------------------------------------------- consumers
    const int cw = wg - 1;                                        // rows 64 cw .. 64 cw + 63 of the tile
    const int q = warp & 3;
    float acc[BN / 2];
#pragma unroll
    for (int r = 0; r < BN / 2; ++r) acc[r] = 0.f;
    // The A fragments of a k-block are read by its MMAs until they retire, so they cannot be rewritten for the next
    // k-block while those are in flight (ptxas serializes the wgmma pipeline if they are).  Each consumer therefore waits
    // for its k-block's MMAs before the next: the other consumer's MMAs keep the tensor pipe busy meanwhile, and the
    // slot goes back to the producer one k-block earlier than with one k-block in flight.
    uint32_t ah[16], al[16];
    for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES, use = i / STAGES;
        tc_mbar_wait(tc_smem_u32(&ready[s]), (uint32_t)(use & 1));      // A and B landed, B's low half written
        tc_mbar_wait(tc_smem_u32(&full[s]), (uint32_t)(use & 1));       // (complete by now) the TMA writes these loads read
        if (threadIdx.x == 128) TC_STAMP(i, 3);
        const uint32_t sa = tc_smem_u32(base + s * STAGE_BYTES);
        tc_load_split_a<A_MN, TF32>(sa, cw, q, lane >> 2, lane & 3, ah, al);
        const uint64_t dB = wg_desc(sa + B_OFF), dBl = wg_desc(sa + B_OFF + B_BYTES);
        wg_fence();
#pragma unroll
        for (int k8 = 0; k8 < TC_BK / 8; ++k8) {
            const uint64_t adv = (uint64_t)((k8 * 32) >> 4);
            if (TF32) {
                WgmmaTf32Rs<BN>::mma(acc, ah + 4 * k8, dB + adv, (i > 0 || k8 > 0) ? 1u : 0u);   // rna . rna
            } else {
                WgmmaTf32Rs<BN>::mma(acc, al + 4 * k8, dB + adv, (i > 0 || k8 > 0) ? 1u : 0u);   // lo . hi
                WgmmaTf32Rs<BN>::mma(acc, ah + 4 * k8, dBl + adv, 1u);                            // hi . lo
                WgmmaTf32Rs<BN>::mma(acc, ah + 4 * k8, dB + adv, 1u);                             // hi . hi
            }
        }
        wg_commit();
        if (threadIdx.x == 128) TC_STAMP(i, 4);
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) tc_mbar_arrive(tc_smem_u32(&empty[s]));
    }

    // -------------------------------------------------------------------- epilogue straight from the accumulator
    float *const Cp = prob ? g.C[1] : g.C[0];     // (a select: indexing the parameter array would copy it to the stack)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + tc_tile_row<A_MN>(cw, q, lane >> 2, h);
        if (m >= g.M) continue;
        float *drow = g.partial ? g.partial + ((int64_t)blockIdx.z * g.M + m) * g.N : Cp + (int64_t)m * g.ldc;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int n = n0 + 8 * j + 2 * (lane & 3);
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if (!g.partial) {
                if (n < g.N) v0 = tc_epilogue(g, Cp, v0, m, n);
                if (n + 1 < g.N) v1 = tc_epilogue(g, Cp, v1, m, n + 1);
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

template <int BN, int STAGES, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmB0,
               const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmB1, GemmTcArgs g) {
    gemm_tc_body<BN, STAGES, A_MN, B_MN, false>(tmA0, tmB0, tmA1, tmB1, g);
}
template <int BN, int STAGES, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_tf32_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmB0,
                    const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmB1, GemmTcArgs g) {
    gemm_tc_body<BN, STAGES, A_MN, B_MN, true>(tmA0, tmB0, tmA1, tmB1, g);
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
// transposing variant: x is rows x cols (ld); outputs are cols x rows (ldo >= rows), tiled through shared memory.
// gridDim.y (at most 65,535) strides over the 32-row tiles, so any row count (K of a weight gradient: T*B) is covered.
__global__ void tc_split_transpose_kernel(const float *__restrict__ x, int64_t ld, int rows, int cols,
                                          float *__restrict__ hi, float *__restrict__ lo, int64_t ldo) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32;
    for (int64_t r0 = (int64_t)blockIdx.y * 32; r0 < ldo; r0 += (int64_t)gridDim.y * 32) {
        for (int i = threadIdx.y; i < 32; i += 8) {
            const int64_t r = r0 + i;
            const int c = c0 + threadIdx.x;
            tile[i][threadIdx.x] = (r < rows && c < cols) ? x[r * ld + c] : 0.f;
        }
        __syncthreads();
        for (int i = threadIdx.y; i < 32; i += 8) {
            const int c = c0 + i;
            const int64_t r = r0 + threadIdx.x;     // output row = c, output col = r
            if (c < cols && r < ldo) {
                const float v = (r < rows) ? tile[threadIdx.x][i] : 0.f;
                const float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
                hi[(int64_t)c * ldo + r] = v;
                if (lo) lo[(int64_t)c * ldo + r] = v - h;
            }
        }
        __syncthreads();
    }
}

// sums the splits of every problem in split order, so a problem's result does not depend on the launch it shared
__global__ void tc_splitk_reduce_kernel(GemmTcArgs g, int problems) {
    const int64_t total = (int64_t)g.M * g.N;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < problems * total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int p = (int)(idx / total);
        const int64_t e = idx - p * total;
        const float *part = g.partial + (int64_t)p * g.splits * total + e;
        float s = 0.f;
        for (int z = 0; z < g.splits; ++z) s += part[(int64_t)z * total];
        const int m = (int)(e / g.N), n = (int)(e % g.N);
        float *const C = p ? g.C[1] : g.C[0];
        C[(int64_t)m * g.ldc + n] = tc_epilogue(g, C, s, m, n);
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

// fp32 2-D tensor map with pitch ld (elements).  K-major (mn = 0): rows x K, box = 32 floats x box_rows, 128B swizzle
// (the layout the wgmma descriptors read).  MN-major (mn = 1): K x rows, box = box_rows floats x 32, 128B-swizzled when
// box_rows is 32 (A: the consumers read their fragments from it) and unswizzled otherwise (B: the producer transposes it).
// Out-of-bounds elements read as 0 either way.
static int make_map(CUtensorMap *m, const float *ptr, int rows, int K, int64_t ld, int box_rows, bool mn) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return set_error(CTCB_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    if (mn) {
        dims[0] = (cuuint64_t)rows; dims[1] = (cuuint64_t)K;
        box[0] = (cuuint32_t)box_rows; box[1] = (cuuint32_t)TC_BK;
    }
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     (mn && box_rows != TC_BK) ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return set_error(CTCB_ECUDA, "cuTensorMapEncodeTiled failed (%d) rows=%d K=%d ld=%lld mn=%d", (int)r, rows, K, (long long)ld, (int)mn);
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

// Splits of one problem of `tiles` output tiles over nkb k-blocks: enough CTAs to cover the SMs, at least 8 k-blocks per
// split, at most 32 splits, and never a chain longer than TC_CHAIN_KB.  A pair of problems keeps the split of one, so
// that each result is bit-identical to its single call (filling whole waves instead would change the summation order).
static int tc_choose_splits(int tiles, int nkb) {
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

// Below these sizes the exact FFMA kernel is used: short contractions (K = 41 / 62) cannot amortise the tensor-core
// pipeline.  The thresholds have not been re-tuned on H100.
constexpr int TC_MIN_K = 128, TC_MIN_M = 32;

// CTCB_GEMM=simt forces the FFMA kernel everywhere
bool gemm_tc_eligible(int M, int N, int K) {
    return !knob(KNOB_GEMM) && get_encode() && M >= TC_MIN_M && N >= 32 && K >= TC_MIN_K;
}

// How an operand reaches the ring.
enum { TC_PATH_KMAJOR = 0,     // TMA reads the caller's K-major array
       TC_PATH_MN = 1,         // TMA reads the caller's MN-major array, the producer transposes in shared memory
       TC_PATH_COPY = 2 };     // a prep kernel re-pitches or transposes it into the workspace first

// TMA needs a 16-byte aligned base and a row pitch that is a multiple of 16 bytes.  CTCB_GEMM_TC_COPY=1: MN-major
// operands go through a transposed copy in the workspace instead of the in-ring transpose; same results at the same
// split, for comparison and timing.
static int tc_operand_path(bool mn_major, const float *p, int64_t ld) {
    if (ld % 4 != 0 || ((uintptr_t)p) % 16 != 0) return TC_PATH_COPY;
    if (mn_major) return knob(KNOB_GEMM_TC_COPY) ? TC_PATH_COPY : TC_PATH_MN;
    return TC_PATH_KMAJOR;
}

struct GemmTcPlan {
    int BN, stages, splits, kb_per_split, ctas, a_path, b_path, problems;
    int tf32;    // TF32 mode (tf32_mode() when planned): gemm_tc_tf32_kernel
};

// The ring depth of a plan.  TF32 mode: as many of its smaller stages as fit in the shared memory of the fp32-faithful
// ring, so both modes hold one CTA per SM alike.
template <int BN, int STAGES>
constexpr int tc_tf32_stages(bool b_mn) {
    return (int)(STAGES * tc_stage_bytes<BN, false, false>() /
                 (b_mn ? tc_stage_bytes<BN, true, true>() : tc_stage_bytes<BN, false, true>()));
}

// The one place that decides how a tensor-core contraction runs: the launcher (run_gemm_tc, run_gemm_tc_pair) and
// ctcb_debug_gemm_plan both call it.  problems = 2 asks for a pair in one launch; a pair with an operand that needs a
// copy runs as two single launches (problems = 1 in the plan).
static void gemm_tc_plan(int transA, int transB, int M, int N, int K, const float *A, int64_t lda, const float *B,
                         int64_t ldb, int problems, GemmTcPlan *p) {
    p->BN = tc_pick_bn(N);
    p->stages = p->BN == 64 ? 4 : 3;     // 192 KB of ring either way: 4 stages of 48 KB (64-wide) or 3 of 64 KB
    p->a_path = tc_operand_path(transA != 0, A, lda);
    p->b_path = tc_operand_path(transB == 0, B, ldb);
    p->tf32 = tf32_mode();
    if (p->tf32) {
        const bool bm = p->b_path == TC_PATH_MN;
        p->stages = p->BN == 64 ? tc_tf32_stages<64, 4>(bm) : tc_tf32_stages<128, 3>(bm);
    }
    p->problems = (problems == 2 && p->a_path != TC_PATH_COPY && p->b_path != TC_PATH_COPY) ? 2 : 1;
    const int tiles = ((M + TC_BM - 1) / TC_BM) * ((N + p->BN - 1) / p->BN);
    const int nkb = (K + TC_BK - 1) / TC_BK;
    const int splits = tc_choose_splits(tiles, nkb);
    p->kb_per_split = (nkb + splits - 1) / splits;
    p->splits = (nkb + p->kb_per_split - 1) / p->kb_per_split;
    p->ctas = p->problems * tiles * p->splits;
}

static size_t tc_partial_bytes(int M, int N, int splits, int problems) {
    return splits > 1 ? (size_t)problems * splits * M * N * sizeof(float) : 0;
}

// Worst case over operand layouts: room for copies of both operands and the partials of a single launch.
size_t gemm_tc_workspace_bytes(int M, int N, int K) {
    const int64_t Kp = pad4(K);
    size_t prep = ((size_t)M * Kp + (size_t)N * Kp) * sizeof(float);
    GemmTcPlan p;
    gemm_tc_plan(0, 1, M, N, K, nullptr, 0, nullptr, 0, 1, &p);
    return align_up(prep, 256) + align_up(tc_partial_bytes(M, N, p.splits, 1), 256) + 1024;
}

// A pair either shares a launch without copies (partials of both problems) or runs as two single launches.
size_t gemm_tc_pair_workspace_bytes(int M, int N, int K) {
    GemmTcPlan p;
    gemm_tc_plan(0, 1, M, N, K, nullptr, 0, nullptr, 0, 2, &p);
    const size_t pair = align_up(tc_partial_bytes(M, N, p.splits, 2), 256) + 1024;
    const size_t single = gemm_tc_workspace_bytes(M, N, K);
    return pair > single ? pair : single;
}

template <int BN, int STAGES, bool A_MN, bool B_MN, bool TF32>
static int launch_tc(const CUtensorMap *tA, const CUtensorMap *tB, const GemmTcArgs &g, int ctas_z, cudaStream_t st) {
    constexpr size_t smem = (size_t)STAGES * tc_stage_bytes<BN, B_MN, TF32>() + 3 * STAGES * 8 + 1024;
    static_assert(smem <= 227 * 1024, "stage ring exceeds the shared memory of a block");
    void (*kernel)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, GemmTcArgs);
    if constexpr (TF32) kernel = gemm_tc_tf32_kernel<BN, STAGES, A_MN, B_MN>;
    else kernel = gemm_tc_kernel<BN, STAGES, A_MN, B_MN>;
    CTCB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((g.N + BN - 1) / BN, (g.M + TC_BM - 1) / TC_BM, ctas_z);
    kernel<<<grid, TC_THREADS, smem, st>>>(tA[0], tB[0], tA[1], tB[1], g);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

template <int BN, int STAGES>
static int launch_tc_paths(const GemmTcPlan &p, const CUtensorMap *tA, const CUtensorMap *tB, const GemmTcArgs &g,
                           cudaStream_t st) {
    const int z = p.problems * p.splits;
    const bool am = p.a_path == TC_PATH_MN, bm = p.b_path == TC_PATH_MN;
    if (p.tf32) {
        constexpr int SK = tc_tf32_stages<BN, STAGES>(false), SM = tc_tf32_stages<BN, STAGES>(true);
        if (am && bm) return launch_tc<BN, SM, true, true, true>(tA, tB, g, z, st);
        if (am) return launch_tc<BN, SK, true, false, true>(tA, tB, g, z, st);
        if (bm) return launch_tc<BN, SM, false, true, true>(tA, tB, g, z, st);
        return launch_tc<BN, SK, false, false, true>(tA, tB, g, z, st);
    }
    if (am && bm) return launch_tc<BN, STAGES, true, true, false>(tA, tB, g, z, st);
    if (am) return launch_tc<BN, STAGES, true, false, false>(tA, tB, g, z, st);
    if (bm) return launch_tc<BN, STAGES, false, true, false>(tA, tB, g, z, st);
    return launch_tc<BN, STAGES, false, false, false>(tA, tB, g, z, st);
}

// One launch (and, with splits, one reduce) of p.problems problems that share shape, pitches, alpha and beta.
// A/B/C: per problem; operands whose path is TC_PATH_COPY must already have been replaced by their copies.
static int run_tc_plan(const GemmTcPlan &p, int M, int N, int K, float alpha, const float *const *A, int64_t lda,
                       const float *const *B, int64_t ldb, float beta, float *const *C, int64_t ldc, const float *bias,
                       int relu, const float *mask_src, float *part, cudaStream_t st) {
    GemmTcArgs g;
    g.M = M; g.N = N; g.K = K; g.ldc = ldc; g.alpha = alpha; g.beta = beta; g.bias = bias; g.relu = relu; g.mask = mask_src;
    g.C[0] = C[0]; g.C[1] = p.problems > 1 ? C[1] : C[0];
    g.trace = nullptr;
    if (knob(KNOB_GEMM_TRACE)) {
        if (!g_gemm_trace) cudaMalloc(&g_gemm_trace, 64 * 8 * sizeof(unsigned long long));
        g.trace = g_gemm_trace;
    }
    g.kb_per_split = p.kb_per_split;
    g.splits = p.splits;
    g.partial = p.splits > 1 ? part : nullptr;

    CUtensorMap tA[2], tB[2];
    int rc;
    for (int q = 0; q < p.problems; ++q) {
        const bool a_mn = p.a_path == TC_PATH_MN;
        if ((rc = make_map(&tA[q], A[q], M, K, lda, a_mn ? 32 : TC_BM, a_mn)) != CTCB_OK) return rc;
        if ((rc = make_map(&tB[q], B[q], N, K, ldb, p.BN, p.b_path == TC_PATH_MN)) != CTCB_OK) return rc;
    }
    if (p.problems == 1) { tA[1] = tA[0]; tB[1] = tB[0]; }
    rc = (p.BN == 64) ? launch_tc_paths<64, 4>(p, tA, tB, g, st) : launch_tc_paths<128, 3>(p, tA, tB, g, st);
    if (rc != CTCB_OK) return rc;
    if (p.splits > 1) {
        const int64_t total = (int64_t)p.problems * M * N;
        int blocks = (int)((total + 255) / 256);
        if (blocks > 4 * num_sms()) blocks = 4 * num_sms();
        tc_splitk_reduce_kernel<<<blocks, 256, 0, st>>>(g, p.problems);
        CTCB_LAUNCH_CHECK();
    }
    return CTCB_OK;
}

// Same contract as ctcb_gemm_f32; ws must hold gemm_tc_workspace_bytes(M, N, K).
int run_gemm_tc(int transA, int transB, int M, int N, int K, float alpha, const float *A, int64_t lda, const float *B,
                int64_t ldb, float beta, float *C, int64_t ldc, const float *bias, int relu, const float *mask_src,
                void *ws, size_t ws_bytes, cudaStream_t st) {
    if (ws_bytes < gemm_tc_workspace_bytes(M, N, K)) return set_error(CTCB_ENOMEM, "run_gemm_tc: workspace too small");
    GemmTcPlan p;
    gemm_tc_plan(transA, transB, M, N, K, A, lda, B, ldb, 1, &p);
    const int64_t Kp = pad4(K);
    float *prep = (float *)ws;
    size_t prep_bytes = 0;
    auto ew_grid = [](int64_t n) { int64_t b = (n + 255) / 256; const int cap = 16 * num_sms(); return (int)(b > cap ? cap : (b < 1 ? 1 : b)); };
    // an operand that TMA cannot read in place becomes rows x Kp, K-major, in the workspace
    auto copy = [&](const float *X, int64_t ld, int rows, bool mn_major, const float **use, int64_t *ld_use) -> int {
        float *dst = prep + prep_bytes / sizeof(float);
        if (mn_major)
            tc_split_transpose_kernel<<<dim3((rows + 31) / 32, (K + 31) / 32 < 65535 ? (K + 31) / 32 : 65535), dim3(32, 8), 0,
                                        st>>>(X, ld, K, rows, dst, nullptr, Kp);
        else
            tc_split_kernel<<<ew_grid((int64_t)rows * Kp), 256, 0, st>>>(X, ld, rows, K, dst, nullptr, Kp);
        CTCB_LAUNCH_CHECK();
        prep_bytes += (size_t)rows * Kp * sizeof(float);
        *use = dst; *ld_use = Kp;
        return CTCB_OK;
    };
    const float *Ause = A, *Buse = B;
    int64_t lda_use = lda, ldb_use = ldb;
    int rc;
    if (p.a_path == TC_PATH_COPY && (rc = copy(A, lda, M, transA != 0, &Ause, &lda_use)) != CTCB_OK) return rc;
    if (p.b_path == TC_PATH_COPY && (rc = copy(B, ldb, N, transB == 0, &Buse, &ldb_use)) != CTCB_OK) return rc;
    float *part = (float *)((char *)ws + align_up(prep_bytes, 256));
    return run_tc_plan(p, M, N, K, alpha, &Ause, lda_use, &Buse, ldb_use, beta, &C, ldc, bias, relu, mask_src, part, st);
}

// Two contractions of one shape in one launch: C_q = alpha op(A_q) op(B_q) + beta C_q, q = 0, 1.  Falls back to two
// run_gemm_tc calls when an operand needs a copy.  ws must hold gemm_tc_pair_workspace_bytes(M, N, K).
int run_gemm_tc_pair(int transA, int transB, int M, int N, int K, float alpha, const float *const *A, int64_t lda,
                     const float *const *B, int64_t ldb, float beta, float *const *C, int64_t ldc, void *ws,
                     size_t ws_bytes, cudaStream_t st) {
    if (ws_bytes < gemm_tc_pair_workspace_bytes(M, N, K)) return set_error(CTCB_ENOMEM, "run_gemm_tc_pair: workspace too small");
    GemmTcPlan p, p1;
    gemm_tc_plan(transA, transB, M, N, K, A[0], lda, B[0], ldb, 2, &p);
    gemm_tc_plan(transA, transB, M, N, K, A[1], lda, B[1], ldb, 2, &p1);
    if (p.problems == 2 && p1.problems == 2)
        return run_tc_plan(p, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, nullptr, 0, nullptr, (float *)ws, st);
    for (int q = 0; q < 2; ++q) {
        const int rc = run_gemm_tc(transA, transB, M, N, K, alpha, A[q], lda, B[q], ldb, beta, C[q], ldc, nullptr, 0,
                                   nullptr, ws, ws_bytes, st);
        if (rc != CTCB_OK) return rc;
    }
    return CTCB_OK;
}

}  // namespace ctcb

// The plan a contraction runs on (include/ctcb200.h); A and B are only inspected for their alignment.
extern "C" int ctcb_debug_gemm_plan(int transA, int transB, int M, int N, int K, const float *A, int64_t lda,
                                    const float *B, int64_t ldb, int problems, int32_t *out) {
    if (!out) return ctcb::set_error(CTCB_EINVAL, "ctcb_debug_gemm_plan: null output");
    if (problems != 1 && problems != 2) return ctcb::set_error(CTCB_EINVAL, "ctcb_debug_gemm_plan: problems must be 1 or 2");
    for (int i = 0; i < 8; ++i) out[i] = 0;
    if (M <= 0 || N <= 0) { out[7] = 1; return CTCB_OK; }      // nothing runs
    if (!ctcb::gemm_tc_eligible(M, N, K)) {                     // FFMA kernel, with room for its partials
        ctcb::GemmSimtPlan s;
        ctcb::gemm_simt_plan(M, N, K, A, lda, B, ldb, SIZE_MAX, &s);
        const int32_t v[8] = {0, 128, 0, s.splits, s.ctas, s.vec, 0, 1};
        for (int i = 0; i < 8; ++i) out[i] = v[i];
        return CTCB_OK;
    }
    ctcb::GemmTcPlan p;
    ctcb::gemm_tc_plan(transA, transB, M, N, K, A, lda, B, ldb, problems, &p);
    const int32_t v[8] = {1, p.BN, p.stages, p.splits, p.ctas, p.a_path, p.b_path, p.problems};
    for (int i = 0; i < 8; ++i) out[i] = v[i];
    return CTCB_OK;
}

extern "C" int ctcb_debug_gemm_plan_tf32(int transA, int transB, int M, int N, int K, const float *A, int64_t lda,
                                         const float *B, int64_t ldb, int problems, int32_t *out) {
    ctcb::Tf32Scope tf32(1);
    return ctcb_debug_gemm_plan(transA, transB, M, N, K, A, lda, B, ldb, problems, out);
}

// Diagnostic: the per-k-block clock stamps of CTA (0,0,0) of the last tensor-core GEMM (CTCB_GEMM_TRACE=1):
// [64][8] = {TMA issued, tiles landed, B's lo written, consumers saw it, MMAs issued}.  Returns 0 when tracing is off.
extern "C" int ctcb_debug_gemm_trace(unsigned long long *host_out) {
    if (!ctcb::g_gemm_trace || !host_out) return 0;
    if (cudaMemcpy(host_out, ctcb::g_gemm_trace, 64 * 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
    return 64;
}
