// sweep_tc.cu -- the temporal-layer recurrences on the Hopper tensor cores (H >= 1024: C3 / C4).
//
// Same arithmetic as sweep.cu / sweep_cluster.cu (reference loops ctc_fast/nnets/brnnet.py:144-152 forward,
// :208-224 BPTT): per time step and direction  S_t = f(pre_t + S_{t-1} . W^T)  over ALL utterances of the batch.
// At H >= 1024 the recurrent matrix no longer fits the register files (sweep_cluster.cu) and the general kernel
// (sweep.cu) re-reads it per 8-utterance tile; here a step is one fp32-faithful (3xTF32, as gemm_tc.cu) tensor-core
// contraction  D[units x utterances] = W[units x H] . S_{t-1}[utterances x H]^T  spread over the device:
//
//   * work split: M tiles of 128 output units x CS K-slices (H/CS inputs each) x NS utterance splits x 2 directions;
//     one persistent CTA per SM for the whole sweep, so every CTA must be co-resident: CS = 4, 2 or 1, the largest
//     whose clusters the device can hold at once (at H = 2048 two directions need 32 clusters of 4, which a 132-SM
//     H100 cannot place; 64 clusters of 2 it can);
//   * the CS K-slices of an (M tile, utterance split, direction) form a CLUSTER: each CTA accumulates its partial
//     product in registers (two warpgroups, 64 units each, wgmma .tf32; hi AND lo halves of both operands arrive by
//     TMA in a 128B-swizzled ring: W's are prepared once per launch, the state's are written by the previous step's
//     epilogue, so no thread touches the operands), copies it to its own shared memory, and after one cluster barrier
//     CTA r sums the four partials of ITS quarter of the utterances through distributed shared memory
//     (ld.shared::cluster), adds pre_t, applies clip / mask and writes S_t -- a deterministic split-K reduction
//     that never touches global memory;
//   * S_t goes to HBM/L2 anyway (the layer's output); the next step's B operand is TMA-loaded from there, so the only
//     device-wide synchronisation is ONE counter barrier per step and (direction, utterance split);
//   * W is streamed from L2 every step (hi + lo of both directions: 16 MB at H = 1024, 64 MB at H = 2048, against the
//     50 MB L2 of an H100); the stream is hidden behind the MMAs whenever the batch is large enough.
// Scratch: the (hi, lo) stacks of W (W^T for BPTT) for both directions and the two-slot ring of state low halves.
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <stdlib.h>

namespace ctcb {

constexpr int STC_THREADS = 288;     // warps 0-7: two consumer warpgroups; warp 8: TMA producer
constexpr int STC_BM = 128;          // output units per CTA
constexpr int STC_BK = 32;           // floats per k-block (one 128-byte swizzle span)
constexpr uint32_t STC_A_BYTES = STC_BM * STC_BK * 4;

struct SweepTcArgs {
    int mode, T, B, H;
    const int32_t *Tlen;
    const float *pre;
    float *out[2];
    float *ring[2];           // [2][B][H] per direction: low halves (x - tf32(x)) of the last two states
    const float *act[2];
    float maxAct;
    unsigned int *err;        // [0]: set to 3 when a wait timed out (results invalid, never a hang)
    unsigned int *counters;   // [ndir * NS] step counters, zeroed before launch
    int ndir, MT, NS;
    int cs;                   // K-slices = cluster size (4, 2 or 1)
    int nkb;                  // k-blocks per K-slice = H / cs / 32
    int stages;
    uint32_t stage_bytes;     // 2 * STC_A_BYTES + 2 * NP * 128
    int partial_own;          // 1: the partial product has its own shared-memory region (W prefetch across steps)
    unsigned long long *trace;   // optional (CTCB_SWEEP_TRACE): [64 steps][16] SM clock stamps of CTA (0,0,0)
};
constexpr int STC_TRACE_STEPS = 64;
#define STC_STAMP(slot)                                                                                         \
    do {                                                                                                        \
        if (a.trace && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && s < STC_TRACE_STEPS)           \
            a.trace[s * 16 + (slot)] = (unsigned long long)clock64();                                           \
    } while (0)

// ---------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t stc_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void stc_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void stc_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool stc_mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait: after ~1 s (or once any thread of the CTA has given up) report through *err and stop waiting, so a
// protocol bug or a lost peer becomes an error flag, never a hung GPU.
__device__ __forceinline__ void stc_mbar_wait(uint32_t bar, uint32_t parity, volatile int *dead, unsigned int *err) {
    if (stc_mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!stc_mbar_try_wait(bar, parity)) {
        if (*dead) return;
        if (clock64() - t0 > 2000000000LL) {
            *dead = 1;
            atomicExch(err, 3u);
            return;
        }
    }
}
// One lane of a converged warp: the producer warp runs its loop warp-uniform and issues from the elected lane.
__device__ __forceinline__ bool stc_elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void stc_tma_3d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void stc_tma_4d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void stc_prefetch_map(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void stc_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t stc_map_to_cta(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ float4 stc_ld_cluster_f4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}
// named barrier of the 256 consumer threads (barrier 0 is __syncthreads)
__device__ __forceinline__ void stc_consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------
// grid = (cs K-slices [cluster], MT * NS, ndir); NP = utterances per split (the wgmma N, a multiple of 32); 9 warps:
//   warp 8 (elected lane) : TMA producer -- W (hi+lo stack, one 3-D box) as soon as a ring slot is free, even across
//                   the step boundary; the state tiles (hi and lo, one 4-D box) once the counter barrier of the
//                   previous step has been seen;
//   warps 0-7     : two warpgroups, units 0..63 / 64..127 of the tile: 4 k-steps x 3 wgmma per k-block, the
//                   accumulator in registers; then registers -> shared partial, cluster barrier, split-K reduction over
//                   DSMEM, epilogue (state, its low half for the next step, one counter arrival per CTA).
// There is no generic-proxy write into the operand ring: both halves of both operands arrive by TMA.
// ---------------------------------------------------------------------------------------------------
template <int NP>
__global__ void __launch_bounds__(STC_THREADS, 1)
sweep_tc_kernel(const __grid_constant__ CUtensorMap tmW0, const __grid_constant__ CUtensorMap tmW1,
                const __grid_constant__ CUtensorMap tmR0, const __grid_constant__ CUtensorMap tmR1, SweepTcArgs a) {
    extern __shared__ __align__(1024) uint8_t stc_smem[];
    uint8_t *base = (uint8_t *)(((uintptr_t)stc_smem + 1023) & ~(uintptr_t)1023);
    const int STAGES = a.stages;
    const uint32_t stage_bytes = a.stage_bytes;
    constexpr uint32_t B_BYTES = (uint32_t)NP * 128u;
    constexpr uint32_t s_off = 2 * STC_A_BYTES;                      // where the state tiles sit inside a stage
    uint8_t *after_ring = base + (size_t)STAGES * stage_bytes;
    // the partial product [NP][128] has a region of its own when it fits (then W tiles of the NEXT step may land in
    // the ring while peers still read this CTA's partial); otherwise it aliases the ring and nothing is prefetched
    float *partial = reinterpret_cast<float *>(a.partial_own ? after_ring : base);
    uint64_t *bars = reinterpret_cast<uint64_t *>(after_ring + (a.partial_own ? (size_t)NP * 512 : 0));
    uint64_t *fullW = bars, *fullS = bars + 8, *empty = bars + 16;
    volatile int *dead = reinterpret_cast<volatile int *>(bars + 24);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rank = blockIdx.x;                                      // K-slice = rank in cluster
    const int mt = blockIdx.y % a.MT, ns = blockIdx.y / a.MT;
    const int dir = blockIdx.z;
    const int B = a.B, T = a.T, H = a.H, nkb = a.nkb;
    const int m0 = mt * STC_BM;
    const int b_lo = ns * NP;
    const int Nc = NP / a.cs;                                         // utterance columns this CTA finalises (<= 64)
    const bool bptt = (a.mode == 1);
    const bool ascending = (dir == 0) != bptt;
    const CUtensorMap *tmW = dir ? &tmW1 : &tmW0;
    // the state as the next step reads it: ring[parity][plane: 0 = value, 1 = low half][B][H]; ONE 4-D box fetches both
    // planes of a k-block
    const CUtensorMap *tmR = dir ? &tmR1 : &tmR0;
    float *out = a.out[dir];
    float *ring = a.ring[dir];                                        // [2 parities][2 planes][B][H]
    const float *act = a.act[dir];
    unsigned int *ctr = a.counters + (dir * a.NS + ns);
    const unsigned int domain = (unsigned int)(a.cs * a.MT);          // CTAs that share this counter

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            stc_mbar_init(stc_smem_u32(&fullW[s]), 1);
            stc_mbar_init(stc_smem_u32(&fullS[s]), 1);
            stc_mbar_init(stc_smem_u32(&empty[s]), 8);                // one arrival per consumer warp
        }
        *dead = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        stc_prefetch_map(tmW);
        stc_prefetch_map(tmR);
    }
    __syncthreads();
    stc_cluster_sync();

    // epilogue role (warps 0-7): warp w takes columns c = w, w + 8, ... < Nc of this CTA's quarter; lane l owns units 4l..4l+3
    const int j4 = m0 + 4 * lane;
    // ring bookkeeping in units of k-block jobs g = (s - 1) * nkb + i (s = 1 .. T-1): stage g % STAGES, use g / STAGES
    uint32_t gW = 0;              // producer: next job whose W tiles have not been requested yet

    // issue the W tiles (hi + lo in one 3-D box) of job g; the caller guarantees the slot is free
    auto issue_W = [&](uint32_t g) {
        const int st = (int)(g % (uint32_t)STAGES);
        const uint32_t fb = stc_smem_u32(&fullW[st]);
        stc_mbar_expect_tx(fb, 2 * STC_A_BYTES);
        const int i = (int)(g % (uint32_t)nkb);
        stc_tma_3d(stc_smem_u32(base + (size_t)st * stage_bytes), tmW, fb, (rank * nkb + i) * STC_BK, m0, 0);   // both planes
    };

    for (int s = 0; s < T; ++s) {
        const int t = ascending ? s : T - 1 - s;
        // operands of the epilogue that do not depend on the recurrence: loaded once the MMAs of the step are done (they
        // would otherwise hold 72 registers across the MMA loop), so that they travel during the cluster barrier
        float4 pre_v[8], act_v[8];
        int Tb[8];
        auto load_epilogue_operands = [&]() {
#pragma unroll
            for (int ci = 0; ci < 8; ++ci) {
                const int c = warp + 8 * ci;
                const int b = b_lo + rank * Nc + c;
                pre_v[ci] = make_float4(0.f, 0.f, 0.f, 0.f);
                act_v[ci] = pre_v[ci];
                Tb[ci] = 0;
                if (warp < 8 && c < Nc && b < B) {
                    const int64_t o = ((int64_t)t * B + b) * H + j4;
                    pre_v[ci] = __ldg(reinterpret_cast<const float4 *>(a.pre + o));
                    if (bptt) act_v[ci] = __ldg(reinterpret_cast<const float4 *>(act + o));
                    Tb[ci] = __ldg(a.Tlen + b);
                }
            }
        };
        if (s == 0) load_epilogue_operands();
        if (s > 0) {
            const uint32_t g0 = (uint32_t)(s - 1) * (uint32_t)nkb, g1 = g0 + (uint32_t)nkb;
            if (warp == 8) {
                // ---------------------------------------------------- TMA producer (whole warp, elected issue)
                const bool leader = stc_elect_one();
                if (leader) STC_STAMP(0);
                const unsigned int target = domain * (unsigned int)s;
                if (leader) {
                    unsigned int v;
                    const long long t0 = clock64();
                    do {
                        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
                        if (v >= target || *dead) break;
                        if (clock64() - t0 > 2000000000LL) { *dead = 1; atomicExch(a.err, 3u); break; }
                    } while (true);
                    asm volatile("fence.proxy.async;" ::: "memory");  // peers' generic-proxy stores -> this CTA's TMA reads
                    STC_STAMP(1);
                }
                __syncwarp();
                for (uint32_t g = g0; g < g1; ++g) {
                    const int st = (int)(g % (uint32_t)STAGES);
                    const uint32_t use = g / (uint32_t)STAGES;
                    const bool need_w = g >= gW;
                    if (need_w && use > 0) stc_mbar_wait(stc_smem_u32(&empty[st]), (use - 1) & 1, dead, a.err);
                    if (need_w) gW = g + 1;
                    const uint32_t fb = stc_smem_u32(&fullS[st]);
                    const uint32_t sdst = stc_smem_u32(base + (size_t)st * stage_bytes + s_off);
                    const int kc = (rank * nkb + (int)(g % (uint32_t)nkb)) * STC_BK;
                    if (leader) {
                        if (need_w) issue_W(g);
                        stc_mbar_expect_tx(fb, 2 * B_BYTES);
                        stc_tma_4d(sdst, tmR, fb, kc, b_lo, 0, (s - 1) & 1);
                    }
                    __syncwarp();
                }
                if (leader) STC_STAMP(2);
                if (a.partial_own && s + 1 < T) {
                    // request the first W tiles of the NEXT step as their slots come free -- they travel while this
                    // CTA finishes its MMAs, reduces, stores and waits at the counter barrier
                    const uint32_t gend = g1 + (uint32_t)((nkb < STAGES) ? nkb : STAGES);
                    for (uint32_t g = g1; g < gend; ++g) {
                        const int st = (int)(g % (uint32_t)STAGES);
                        const uint32_t use = g / (uint32_t)STAGES;
                        if (use > 0) stc_mbar_wait(stc_smem_u32(&empty[st]), (use - 1) & 1, dead, a.err);
                        if (leader) issue_W(g);
                        __syncwarp();
                    }
                    gW = gend;
                }
                __syncwarp();
            } else {
                // ---------------------------------------------------- consumers: warpgroup cw, units 64 cw .. 64 cw + 63
                const int cw = warp >> 2;
                float acc[NP / 2];        // per step: dead once the partial is written
#pragma unroll
                for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
                for (uint32_t g = g0; g < g1; ++g) {
                    const int st = (int)(g % (uint32_t)STAGES);
                    const uint32_t use = g / (uint32_t)STAGES;
                    stc_mbar_wait(stc_smem_u32(&fullW[st]), use & 1, dead, a.err);
                    stc_mbar_wait(stc_smem_u32(&fullS[st]), use & 1, dead, a.err);
                    if (tid == 0 && g == g0) STC_STAMP(3);
                    const uint32_t sa = stc_smem_u32(base + (size_t)st * stage_bytes);
                    const uint64_t dA = wg_desc(sa + (uint32_t)cw * (64 * 128)), dAl = wg_desc(sa + STC_A_BYTES + (uint32_t)cw * (64 * 128));
                    const uint64_t dB = wg_desc(sa + s_off), dBl = wg_desc(sa + s_off + B_BYTES);
                    wg_fence();
#pragma unroll
                    for (int k8 = 0; k8 < STC_BK / 8; ++k8) {
                        const uint64_t adv = (uint64_t)((k8 * 32) >> 4);
                        WgmmaTf32<NP>::mma(acc, dAl + adv, dB + adv, (g > g0 || k8 > 0) ? 1u : 0u);   // lo . hi
                        WgmmaTf32<NP>::mma(acc, dA + adv, dBl + adv, 1u);                           // hi . lo
                        WgmmaTf32<NP>::mma(acc, dA + adv, dB + adv, 1u);                            // hi . hi
                    }
                    wg_commit();
                    // the previous job's MMAs are complete once at most this one is outstanding: release its slot
                    wg_wait<1>();
                    if (g > g0) {
                        __syncwarp();
                        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(stc_smem_u32(&empty[(g - 1) % (uint32_t)STAGES])) : "memory");
                    }
                }
                wg_wait<0>();
                __syncwarp();
                if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(stc_smem_u32(&empty[(g1 - 1) % (uint32_t)STAGES])) : "memory");
                if (tid == 0) STC_STAMP(4);
                // ---------------------------------------------------- partial product: registers -> shared
                if (!a.partial_own) stc_consumer_sync();     // the partial aliases the ring: both warpgroups are done with it
                const int q = warp & 3;
                const int u0 = 64 * cw + 16 * q + (lane >> 2);
#pragma unroll
                for (int i = 0; i < NP / 2; ++i) {
                    const int unit = u0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
                    partial[col * STC_BM + unit] = acc[i];
                }
            }
            load_epilogue_operands();
            if (tid == 64) STC_STAMP(6);
            __syncthreads();         // implied by the cluster barrier below; stated for tools that only model CTA barriers
            stc_cluster_sync();      // all four partials of this (M tile, split) are in shared memory
            if (tid == 64) STC_STAMP(7);
        }
        // ------------------------------------------------------------ split-K reduction over DSMEM + epilogue
        float *ring_s = ring + (size_t)(s & 1) * 2 * B * H;             // plane 0: the state, plane 1: its low half
#pragma unroll
        for (int ci = 0; ci < 8; ++ci) {
            const int c = warp + 8 * ci;
            if (warp >= 8 || c >= Nc) continue;
            const int b = b_lo + rank * Nc + c;
            float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
            if (s > 0) {
                const uint32_t local = stc_smem_u32(partial + (rank * Nc + c) * STC_BM + 4 * lane);
                for (int q = 0; q < a.cs; ++q) {
                    const float4 p = stc_ld_cluster_f4(stc_map_to_cta(local, (uint32_t)q));
                    sum.x += p.x; sum.y += p.y; sum.z += p.z; sum.w += p.w;
                }
            }
            if (b < B) {
                float4 v;
                v.x = pre_v[ci].x + sum.x; v.y = pre_v[ci].y + sum.y; v.z = pre_v[ci].z + sum.z; v.w = pre_v[ci].w + sum.w;
                if (!bptt) {
                    v.x = fminf(fmaxf(v.x, 0.f), a.maxAct); v.y = fminf(fmaxf(v.y, 0.f), a.maxAct);
                    v.z = fminf(fmaxf(v.z, 0.f), a.maxAct); v.w = fminf(fmaxf(v.w, 0.f), a.maxAct);
                } else {
                    v.x = (act_v[ci].x > 0.f && act_v[ci].x < a.maxAct) ? v.x : 0.f;
                    v.y = (act_v[ci].y > 0.f && act_v[ci].y < a.maxAct) ? v.y : 0.f;
                    v.z = (act_v[ci].z > 0.f && act_v[ci].z < a.maxAct) ? v.z : 0.f;
                    v.w = (act_v[ci].w > 0.f && act_v[ci].w < a.maxAct) ? v.w : 0.f;
                }
                if (t >= Tb[ci]) v = make_float4(0.f, 0.f, 0.f, 0.f);
                *reinterpret_cast<float4 *>(out + ((int64_t)t * B + b) * H + j4) = v;
                if (s + 1 < T) {      // the next step's B operands: v again (same tensor map as its low half) and the low half
                    *reinterpret_cast<float4 *>(ring_s + (int64_t)b * H + j4) = v;
                    float4 lo;
                    lo.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xffffe000u);
                    lo.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xffffe000u);
                    lo.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xffffe000u);
                    lo.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xffffe000u);
                    *reinterpret_cast<float4 *>(ring_s + (int64_t)(B + b) * H + j4) = lo;
                }
            }
        }
        // ------------------------------------------------------------ publish S_t: one counter arrival per CTA
        if (tid == 64) STC_STAMP(8);
        if (s + 1 < T) {
            __syncthreads();
            if (tid == 0) {
                STC_STAMP(9);
                // release: the CTA's state stores (ordered before this thread by the barrier above) become visible at
                // device scope before the count does.  The generic->async proxy fence belongs to the READER (after its
                // acquire, before its TMA loads).
                asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(ctr), "r"(1u) : "memory");
                STC_STAMP(10);
            }
        }
    }
    // no CTA may exit while a peer can still read its shared memory
    stc_cluster_sync();
}

// Operand preparation, once per launch: out[0] = W (or W^T for BPTT), out[1] = its low half x - tf32(x); both H x H
// row-major, stacked so that ONE 3-D TMA box fetches the hi and the lo tile of a k-block.
__global__ void stc_prep_kernel(const float *__restrict__ w, float *__restrict__ stack, int H, int transpose) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    float *hi = stack, *lo = stack + (size_t)H * H;
    if (transpose) {
        for (int i = threadIdx.y; i < 32; i += 8) tile[i][threadIdx.x] = w[(int64_t)(r0 + i) * H + c0 + threadIdx.x];
        __syncthreads();
        for (int i = threadIdx.y; i < 32; i += 8) {
            const float v = tile[threadIdx.x][i];
            const int64_t o = (int64_t)(c0 + i) * H + r0 + threadIdx.x;
            hi[o] = v;
            lo[o] = v - __uint_as_float(__float_as_uint(v) & 0xffffe000u);
        }
    } else {
        for (int i = threadIdx.y; i < 32; i += 8) {
            const int64_t o = (int64_t)(r0 + i) * H + c0 + threadIdx.x;
            const float v = w[o];
            hi[o] = v;
            lo[o] = v - __uint_as_float(__float_as_uint(v) & 0xffffe000u);
        }
    }
}

// ---------------------------------------------------------------------------------- host side
typedef CUresult (*StcEncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static StcEncodeFn stc_encode() {
    static StcEncodeFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (StcEncodeFn)p;
        else
            cudaGetLastError();
    }
    return fn;
}

struct StcPlan { int cs, NS, Npad, stages, partial_own; uint32_t stage_bytes; size_t smem; };

static constexpr size_t STC_SMEM_MAX = 208 * 1024;      // ring + partial budget (+ barriers) within the 227 KB per CTA

// co-resident clusters of cs CTAs (the kernel's shared memory does not depend on NP for this question: every plan
// uses about STC_SMEM_MAX, so one CTA per SM)
static int stc_max_clusters(int cs) {
    static int cached[5] = {-1, -1, -1, -1, -1};
    if (cached[cs] >= 0) return cached[cs];
    const size_t smem = STC_SMEM_MAX + 2048;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cs, 64, 2);
    cfg.blockDim = dim3(STC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    int n = 0;
    if (cudaFuncSetAttribute(sweep_tc_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
        cudaOccupancyMaxActiveClusters(&n, sweep_tc_kernel<256>, &cfg) != cudaSuccess) {
        cudaGetLastError();
        n = 0;
    }
    cached[cs] = n;
    if (getenv("CTCB_DEBUG")) fprintf(stderr, "[ctcb] tensor-core sweep: max active clusters of %d CTAs = %d\n", cs, n);
    return n;
}

// Per cluster size, largest first: every CTA of the grid must be co-resident (they meet at the counter barrier), and a
// CTA finalises at most 64 utterance columns (NP / cs <= 64).
static bool stc_plan_cs(int H, int B, int ndir, int cs, StcPlan *p) {
    const int MT = H / STC_BM;
    if ((H / cs) % STC_BK != 0) return false;
    const int maxc = stc_max_clusters(cs);
    if (maxc < ndir * MT) return false;
    int ns_cap = maxc / (ndir * MT);
    static int ns_env = -1;
    if (ns_env < 0) { const char *e = getenv("CTCB_SWEEP_TC_NS"); ns_env = e ? atoi(e) : 0; }
    if (ns_env > 0 && ns_env < ns_cap) ns_cap = ns_env;
    int NS = (B + 15) / 16;                  // never more splits than 16-utterance groups
    if (NS > ns_cap) NS = ns_cap;
    if (NS < 1) NS = 1;
    const int Npad = ((B + NS - 1) / NS + 31) / 32 * 32;   // the wgmma N of the kernel: a multiple of 32 up to 256
    if (Npad > 256 || Npad > 64 * cs) return false;
    p->cs = cs;
    p->NS = (B + Npad - 1) / Npad;           // drop splits that would be empty
    p->Npad = Npad;
    const size_t partial_bytes = (size_t)Npad * 512;
    p->stage_bytes = 2 * STC_A_BYTES + 2 * (uint32_t)Npad * 128u;
    // own region for the partial when at least two ring stages still fit beside it
    p->partial_own = (STC_SMEM_MAX >= partial_bytes + 2 * (size_t)p->stage_bytes) ? 1 : 0;
    int stages = (int)((STC_SMEM_MAX - (p->partial_own ? partial_bytes : 0)) / p->stage_bytes);
    if (stages > 6) stages = 6;
    if (stages < 2) return false;
    if (!p->partial_own && (size_t)stages * p->stage_bytes < partial_bytes) return false;    // the ring must hold the aliased partial
    p->stages = stages;
    p->smem = (size_t)stages * p->stage_bytes + (p->partial_own ? partial_bytes : 0) + 256 + 1024;
    return true;
}

static bool stc_plan(int H, int B, int ndir, StcPlan *p) {
    if (H % 128 != 0 || H < 512 || B < 1) return false;
    for (int cs = 4; cs >= 1; cs >>= 1)
        if (stc_plan_cs(H, B, ndir, cs, p)) {
            if (getenv("CTCB_DEBUG"))
                fprintf(stderr, "[ctcb] tensor-core sweep H=%d B=%d: clusters of %d, %d utterance split(s) of %d\n", H, B, cs, p->NS, p->Npad);
            return true;
        }
    return false;
}

static bool stc_enabled(int H) {
    static int mode = -1;     // CTCB_SWEEP_TC=0 disables, =1 default (H >= 1024), =2 also H = 512
    if (mode < 0) { const char *e = getenv("CTCB_SWEEP_TC"); mode = e ? atoi(e) : 1; }
    if (mode == 0 || !stc_encode()) return false;
    return H >= 1024 || (mode == 2 && H >= 512);
}

// scratch: (hi, lo) stacks of both recurrent matrices, the rings of state low halves, the optional trace
static size_t stc_ws_stack_bytes(int H) { return align_up((size_t)4 * H * H * sizeof(float), 1024); }
static size_t stc_ws_ring_bytes(int H, int B) { return align_up((size_t)8 * B * H * sizeof(float), 1024); }
size_t sweep_tc_workspace_bytes(int H, int B) {
    return stc_ws_stack_bytes(H) + stc_ws_ring_bytes(H, B) + STC_TRACE_STEPS * 16 * 8 + 1024;
}

template <int NP>
static cudaError_t stc_launch(cudaLaunchConfig_t *cfg, const CUtensorMap *tmW, const CUtensorMap *tmR, const SweepTcArgs &a) {
    cudaError_t e = cudaFuncSetAttribute(sweep_tc_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg->dynamicSmemBytes);
    if (e != cudaSuccess) return e;
    return cudaLaunchKernelEx(cfg, sweep_tc_kernel<NP>, tmW[0], tmW[1], tmR[0], tmR[1], a);
}
static cudaError_t stc_launch_np(int np, cudaLaunchConfig_t *cfg, const CUtensorMap *tmW, const CUtensorMap *tmR, const SweepTcArgs &a) {
    switch (np) {
        case 32: return stc_launch<32>(cfg, tmW, tmR, a);
        case 64: return stc_launch<64>(cfg, tmW, tmR, a);
        case 96: return stc_launch<96>(cfg, tmW, tmR, a);
        case 128: return stc_launch<128>(cfg, tmW, tmR, a);
        case 160: return stc_launch<160>(cfg, tmW, tmR, a);
        case 192: return stc_launch<192>(cfg, tmW, tmR, a);
        case 224: return stc_launch<224>(cfg, tmW, tmR, a);
        default: return stc_launch<256>(cfg, tmW, tmR, a);
    }
}

int run_sweep_tc(int mode, int T, int B, int H, const int32_t *Tlen, const float *pre, const float *Wf, const float *Wb,
                 float *outF, float *outB, const float *actF, const float *actB, float maxAct, unsigned int *counters,
                 void *ws, size_t ws_bytes, cudaStream_t st, bool *handled) {
    *handled = false;
    const int ndir = Wb ? 2 : 1;
    StcPlan p;
    if (!stc_enabled(H) || !stc_plan(H, B, ndir, &p)) return CTCB_OK;
    // the plan applies, so the generic kernel is no substitute: a scratch that cannot hold the operand stacks is an error
    if (!ws || ws_bytes < sweep_tc_workspace_bytes(H, B) || (((uintptr_t)ws) & 255))
        return set_error(CTCB_ENOMEM, "tensor-core sweep (H=%d, B=%d) needs %zu bytes of 256-byte aligned scratch, got %zu%s",
                         H, B, sweep_tc_workspace_bytes(H, B), ws_bytes, ws ? "" : " (none)");
    StcEncodeFn enc = stc_encode();
    float *stack = (float *)ws;
    float *ring = (float *)((char *)ws + stc_ws_stack_bytes(H));
    const float *Wd[2] = {Wf, Wb ? Wb : Wf};
    for (int d = 0; d < ndir; ++d) {
        stc_prep_kernel<<<dim3(H / 32, H / 32), dim3(32, 8), 0, st>>>(Wd[d], stack + (size_t)d * 2 * H * H, H, mode == 1 ? 1 : 0);
        CTCB_LAUNCH_CHECK();
    }
    float *outs[2] = {outF, Wb ? outB : outF};
    CUtensorMap tmW[2], tmR[2];
    for (int d = 0; d < 2; ++d) {
        const int dd = (d < ndir) ? d : 0;
        {
            cuuint64_t dims[3] = {(cuuint64_t)H, (cuuint64_t)H, 2};
            cuuint64_t strides[2] = {(cuuint64_t)H * sizeof(float), (cuuint64_t)H * H * sizeof(float)};
            cuuint32_t box[3] = {(cuuint32_t)STC_BK, (cuuint32_t)STC_BM, 2};
            cuuint32_t es[3] = {1, 1, 1};
            CUresult r = enc(&tmW[d], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void *)(stack + (size_t)dd * 2 * H * H), dims, strides, box, es,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) return set_error(CTCB_ECUDA, "sweep_tc: cuTensorMapEncodeTiled(W) failed (%d)", (int)r);
        }
        {
            cuuint64_t dims[4] = {(cuuint64_t)H, (cuuint64_t)B, 2, 2};
            cuuint64_t strides[3] = {(cuuint64_t)H * sizeof(float), (cuuint64_t)B * H * sizeof(float), (cuuint64_t)2 * B * H * sizeof(float)};
            cuuint32_t box[4] = {(cuuint32_t)STC_BK, (cuuint32_t)p.Npad, 2, 1};
            cuuint32_t es[4] = {1, 1, 1, 1};
            CUresult r = enc(&tmR[d], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void *)(ring + (size_t)dd * 4 * B * H), dims, strides, box, es,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) return set_error(CTCB_ECUDA, "sweep_tc: cuTensorMapEncodeTiled(state ring) failed (%d)", (int)r);
        }
    }
    SweepTcArgs a;
    a.mode = mode; a.T = T; a.B = B; a.H = H; a.Tlen = Tlen; a.pre = pre;
    a.out[0] = outs[0]; a.out[1] = outs[1]; a.act[0] = actF; a.act[1] = Wb ? actB : actF; a.maxAct = maxAct;
    a.ring[0] = ring; a.ring[1] = ring + (size_t)(ndir - 1) * 4 * B * H;
    a.err = counters; a.counters = counters + 16;
    a.ndir = ndir; a.MT = H / STC_BM; a.NS = p.NS; a.cs = p.cs; a.nkb = H / p.cs / STC_BK;
    a.stages = p.stages; a.stage_bytes = p.stage_bytes; a.partial_own = p.partial_own;
    a.trace = nullptr;
    {
        static int trace_env = -1;
        if (trace_env < 0) trace_env = getenv("CTCB_SWEEP_TRACE") ? 1 : 0;
        if (trace_env) a.trace = (unsigned long long *)((char *)ws + stc_ws_stack_bytes(H) + stc_ws_ring_bytes(H, B));
    }
    CTCB_CUDA_CHECK(cudaMemsetAsync(a.counters, 0, sizeof(unsigned int) * (size_t)(ndir * p.NS), st));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(p.cs, a.MT * p.NS, ndir);
    cfg.blockDim = dim3(STC_THREADS);
    cfg.dynamicSmemBytes = p.smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = p.cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeCooperative;       // co-residency of all CTAs (they meet at the counter barrier)
    attr[1].val.cooperative = 1;
    cfg.attrs = attr;
    static int coop = -1;     // does this driver accept cluster + cooperative together?  (CTCB_SWEEP_TC_COOP=0: plain cluster launch)
    if (coop < 0) { const char *e = getenv("CTCB_SWEEP_TC_COOP"); if (e && atoi(e) == 0) coop = 0; }
    if (coop != 0) {
        cfg.numAttrs = 2;
        cudaError_t e = stc_launch_np(p.Npad, &cfg, tmW, tmR, a);
        if (e == cudaSuccess) { coop = 1; count_launch(); *handled = true; return CTCB_OK; }
        cudaGetLastError();
        if (coop == 1) return set_error(CTCB_ECUDA, "sweep_tc: launch failed: %s", cudaGetErrorString(e));
        coop = 0;
        if (getenv("CTCB_DEBUG")) fprintf(stderr, "[ctcb] tensor-core sweep: cooperative+cluster launch refused (%s), plain cluster launch\n", cudaGetErrorString(e));
    }
    cfg.numAttrs = 1;         // grid <= one wave of clusters by construction (stc_plan)
    CTCB_CUDA_CHECK(stc_launch_np(p.Npad, &cfg, tmW, tmR, a));
    count_launch();
    *handled = true;
    return CTCB_OK;
}

bool sweep_tc_would_run(int H, int B, int ndir) {
    StcPlan p;
    return stc_enabled(H) && stc_plan(H, B, ndir, &p);
}

}  // namespace ctcb

extern "C" int ctcb_sweep_uses_tensor_cores(int H, int B) { return ctcb::sweep_tc_would_run(H, B, 2) ? 1 : 0; }
