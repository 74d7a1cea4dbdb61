// sweep_cluster.cu -- the temporal-layer recurrences on thread-block clusters (H = 128, 256, 512).
//
// Same arithmetic as sweep.cu (reference loops brnnet.py:144-152 forward, :208-224 BPTT), but the
// hidden state never touches global memory on the serial chain:
//
//   * one CLUSTER of CS = H/64 CTAs per (direction, group of NB utterances); CTA r owns 64 output units and
//     keeps its 64 x H slice of the recurrent matrix in registers for the whole sweep;
//   * every CTA holds the complete previous state of its NB utterances in shared memory, laid out
//     [source CTA][utterance][64 units] so that one CTA's contribution is one contiguous block;
//   * after a step, each CTA pushes its block into the shared memory of all CS CTAs of the cluster with
//     4-byte st.async remote stores; each completes its bytes on the DESTINATION's mbarrier for that source CTA,
//     which is the only inter-CTA synchronisation of the step: a warp starts step s as soon as the one block of
//     step s-1 it reads has landed.  Two state buffers, each with CS barriers (one per source CTA), alternate;
//   * For/Back (dFor/dBack) are still streamed to HBM for the GEMMs that follow, off the chain.
#include "common.cuh"
#include <stdlib.h>

namespace ctcb {

struct SweepClusterArgs {
    int mode, T, B, H;
    const int32_t *Tlen;
    const float *pre;
    const float *W[2];
    float *out[2];
    const float *act[2];
    float maxAct;
    unsigned int *err;      // [0] set to 2 if a barrier wait timed out (never a hang)
    int ndir;               // gridDim.z: 2 = both directions, 1 = forward in time only
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t map_to_cta(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Remote 4-byte store into a cluster peer's shared memory that completes 4 bytes of the peer's mbarrier
// transaction count when it has landed (the consumer's try_wait then orders its reads after the data).
__device__ __forceinline__ void st_async_f32(uint32_t dst_cluster, float v, uint32_t bar_cluster) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
                 ::"r"(dst_cluster), "r"(__float_as_uint(v)), "r"(bar_cluster) : "memory");
}

// a pair of output units times one scalar state value: two FFMAs (each rounded exactly as fma.rn)
__device__ __forceinline__ void ffma_pair(float2 &d, float2 w, float h) {
    d.x = fmaf(w.x, h, d.x);
    d.y = fmaf(w.y, h, d.y);
}

// ---------------------------------------------------------------------------------------------------
// The kernel: 16 warps per CTA, 64 output units per CTA, CS = H/64 CTAs per cluster, NB
// utterances per cluster.  The INPUT dimension is split over the warps, not over the lanes: warp w owns input
// units [w*H/16, (w+1)*H/16) of all 64 output units; lane l owns output units 2l, 2l+1 (H/8 weights per thread
// in registers, one register pair per input unit: (pair of units) x (scalar state)).
// Per warp and step at H = 512, NB = 5:
//   * every lane needs the same slice of the previous state: 40 broadcast LDS.128;
//   * no shuffle reduction: a lane's accumulators are complete over its warp's slice; the 16 per-warp partial
//     sums of an output meet in shared memory (the one CTA barrier of the step), where thread (utterance, unit)
//     adds them, applies clip/mask, stores the state to HBM and sends it to the CS peers with st.async.
//   state layout in every CTA: [buffer 2][source CTA][utterance][unit 64]
// Measured on one H100 80GB HBM3 (power limit 700 W, max SM clock 1980 MHz), tools/sweep_time.py, T = 200, H = 512,
// forward / BPTT in us per step: B = 4 (NB = 1) 0.69 / 0.62, B = 8 (NB = 2) 0.98 / 0.91, B = 16 (NB = 3) 1.24 / 1.21,
// B = 32 (NB = 5) 1.77 / 1.78.  Fit: 0.43 / 0.33 us fixed (wait, barrier, reduction, exchange) + 0.27 / 0.29 us per
// utterance of the cluster, of which 32768 FMA per SM at the FFMA peak (128 per clock) would take 0.13 us.
// One barrier per source CTA instead of one per buffer: B = 32 went from 1.87 / 1.81 to 1.77 / 1.78 (the fit above);
// deciding the mask before the barrier and sending before the HBM store then gave 1.74-1.76 / 1.72-1.73.  Sending the
// state as one 16-byte st.async per lane quad and peer (three shuffles to assemble it) was slower on the same card,
// 2.00 / 1.96 with the single barrier and 1.85 / 1.81 with per-source barriers, so the stores stay 4-byte.
// ---------------------------------------------------------------------------------------------------
template <int KI, int NB>
__global__ void __launch_bounds__(512, 1) sweep_cluster_kernel(SweepClusterArgs a) {
    constexpr int H = 32 * KI;
    constexpr int CS = H / 64;
    constexpr int KW = H / 16;                                           // input units per warp
    constexpr int BLKF = NB * 64;                                        // floats per CTA block
    constexpr uint32_t BLK_BYTES = BLKF * sizeof(float);
    static_assert(KW % 4 == 0 && 64 % KW == 0, "warp slice must not straddle two CTA blocks");
    extern __shared__ __align__(128) float sc_smem[];
    float (*hbuf)[CS * BLKF] = reinterpret_cast<float (*)[CS * BLKF]>(sc_smem);                  // [2][source CTA][utterance][unit]
    float (*red)[16][BLKF] = reinterpret_cast<float (*)[16][BLKF]>(sc_smem + 2 * CS * BLKF);     // [2][16 warps][utterance][unit]
    unsigned long long (*mbar)[CS] = reinterpret_cast<unsigned long long (*)[CS]>(sc_smem + (2 * CS + 32) * BLKF);   // [2][source CTA]

    const int B = a.B, T = a.T;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = blockIdx.x;
    const int dir = blockIdx.z;
    const int b0 = blockIdx.y * NB;
    const float *W = a.W[dir];
    float *out = a.out[dir];
    const float *act = a.act[dir];
    const bool bptt = (a.mode == 1);
    const bool ascending = (dir == 0) != bptt;
    const int j0 = rank * 64;
    const int k0 = warp * KW;

    // w2[k] = weights of output units (2*lane, 2*lane + 1) for input unit k0 + k
    float2 w2[KW];
#pragma unroll
    for (int k = 0; k < KW; ++k) {
        const int j = j0 + 2 * lane, kk = k0 + k;
        w2[k] = bptt ? make_float2(W[(int64_t)kk * H + j], W[(int64_t)kk * H + j + 1])
                     : make_float2(W[(int64_t)j * H + kk], W[(int64_t)(j + 1) * H + kk]);
    }

    // one barrier per (state buffer, source CTA), each expecting one block
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 2 * CS; ++i) mbar_init(smem_u32(&mbar[i / CS][i % CS]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#pragma unroll
        for (int i = 0; i < 2 * CS; ++i) mbar_arrive_expect_tx(smem_u32(&mbar[i / CS][i % CS]), BLK_BYTES);
    }
    cluster_sync_all();

    // epilogue role: thread (eu, ej) = (utterance, unit) for tid < NB*64
    const int eu = tid >> 6, ej = tid & 63;
    const int b = b0 + eu, oj = j0 + ej;
    const bool owner = tid < BLKF;
    const bool valid = owner && (b < B);
    const int Tb = valid ? __ldg(a.Tlen + b) : 0;
    // where this warp's slice of the state sits inside a buffer: source CTA k0/64, offset k0%64.  The warp reads
    // nothing else, so it waits only for that source's barrier and starts while later blocks are still landing.
    const int src = k0 >> 6;
    const int hoff = src * BLKF + (k0 & 63);
    // where this thread's state value goes in every CTA (buffer 0; buffer 1 is CS blocks further), and the barrier
    // of (buffer 0, this CTA) it completes
    const uint32_t dst0 = smem_u32(&hbuf[0][rank * BLKF + tid]);
    const uint32_t dbar0 = smem_u32(&mbar[0][rank]);
    bool dead = false;

    for (int s = 0; s < T; ++s) {
        const int t = ascending ? s : T - 1 - s;
        const int64_t o = ((int64_t)t * B + b) * H + oj;       // (t, b, oj) in pre, act and out
        float pre_v = 0.f, act_v = 0.f;
        if (valid) {
            pre_v = __ldg(a.pre + o);
            if (bptt) act_v = __ldg(act + o);
        }
        bool keep = false;                                        // false: v is masked to 0 (padded frame, BPTT outside (0, maxAct))
        float sum = 0.f;
        if (s > 0) {
            const uint32_t bar = smem_u32(&mbar[s & 1][src]);
            const uint32_t parity = (uint32_t)(((s - 1) >> 1) & 1);
            if (!dead && !mbar_try_wait(bar, parity)) {
                const long long t_start = clock64();
                while (!mbar_try_wait(bar, parity)) {
                    if (clock64() - t_start > 1000000000LL) {   // ~0.5 s: report, then run on without waiting
                        dead = true;
                        atomicExch(a.err, 2u);
                        break;
                    }
                }
            }
            const float *hs = &hbuf[s & 1][hoff];
            float2 acc2[NB];
#pragma unroll
            for (int u = 0; u < NB; ++u) {
#pragma unroll
                for (int q = 0; q < KW / 4; ++q) {
                    const float4 hv = *reinterpret_cast<const float4 *>(hs + u * 64 + 4 * q);   // broadcast
                    if (q == 0) acc2[u] = make_float2(0.f, 0.f);
                    ffma_pair(acc2[u], w2[4 * q], hv.x);
                    ffma_pair(acc2[u], w2[4 * q + 1], hv.y);
                    ffma_pair(acc2[u], w2[4 * q + 2], hv.z);
                    ffma_pair(acc2[u], w2[4 * q + 3], hv.w);
                }
            }
#pragma unroll
            for (int u = 0; u < NB; ++u)
                *reinterpret_cast<float2 *>(&red[s & 1][warp][u * 64 + 2 * lane]) = acc2[u];
            // the mask needs only this step's inputs: decide it while the other warps finish
            keep = valid && t < Tb && (!bptt || (act_v > 0.f && act_v < a.maxAct));
            __syncthreads();            // the only CTA barrier of the step (red is double-buffered)
            // Every warp is past its wait on this step's barriers: arm them for step s + 2.  Reusing buffer s & 1 is
            // safe because every send of step s comes after the step-s __syncthreads.  A peer writes buffer s & 1
            // again with its sends of step s + 1, which follow its step-(s + 1) waits, which need this CTA's block of
            // step s, which this CTA sends only after all its warps have read buffer s & 1 (and so after each
            // barrier s & 1 has completed this step's phase).  Those writes may still land before the arm below:
            // their complete_tx only drives the transaction count negative, and the phase cannot complete while
            // the arm's arrival is pending; the arm then adds BLK_BYTES back and the phase completes at zero.
            if (tid < CS && s + 2 < T) mbar_arrive_expect_tx(smem_u32(&mbar[s & 1][tid]), BLK_BYTES);
            if (owner) {
                float s0 = 0.f, s1 = 0.f;
#pragma unroll
                for (int w = 0; w < 16; w += 2) { s0 += red[s & 1][w][tid]; s1 += red[s & 1][w + 1][tid]; }
                sum = s0 + s1;
            }
        }
        if (s == 0) keep = valid && t < Tb && (!bptt || (act_v > 0.f && act_v < a.maxAct));
        float v = pre_v + sum;
        if (!bptt) v = fminf(fmaxf(v, 0.f), a.maxAct);
        v = keep ? v : 0.f;
        if (owner && s + 1 < T) {
            // hand the new state to every CTA of the cluster (this one included): one remote 4-byte store per
            // peer, each completing 4 bytes on the peer's barrier of (step s + 1, this CTA).  Invalid owners send
            // their zeros too: the barrier expects a whole block.  The sends are the serial chain of the sweep,
            // so they go out before the HBM store.
            const uint32_t nbo = (uint32_t)((s + 1) & 1);
            const uint32_t dst = dst0 + nbo * (uint32_t)(CS * BLK_BYTES);
            const uint32_t dbar = dbar0 + nbo * (uint32_t)(CS * sizeof(unsigned long long));
#pragma unroll
            for (int c = 0; c < CS; ++c) st_async_f32(map_to_cta(dst, (uint32_t)c), v, map_to_cta(dbar, (uint32_t)c));
        }
        if (valid) out[o] = v;
    }
    cluster_sync_all();
}

// state buffers + partial sums + 2 x CS mbarriers
static constexpr size_t cluster_smem_bytes(int KI, int NB) {
    return sizeof(float) * (size_t)(2 * (KI / 2) + 32) * (size_t)(NB * 64) + 2 * (KI / 2) * sizeof(unsigned long long);
}

template <int KI, int NB>
static int launch_cluster_nb(const SweepClusterArgs &a, int ntiles, cudaStream_t st) {
    auto kern = sweep_cluster_kernel<KI, NB>;
    constexpr int CS = KI / 2;
    constexpr size_t SMEM = cluster_smem_bytes(KI, NB);
    static bool attr_set = false;
    if (!attr_set) {
        CTCB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
        attr_set = true;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(CS, ntiles, a.ndir);
    cfg.blockDim = dim3(512);
    cfg.dynamicSmemBytes = SMEM;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    // the serial chain of the step: its clusters are placed before any pending CTA of a lower-priority stream (the
    // weight gradients that run next to the BPTT sweep, brnn.cu).  A launch attribute, so a captured graph keeps it.
    attr[1].id = cudaLaunchAttributePriority;
    attr[1].val.priority = stream_priority_greatest();
    cfg.attrs = attr;
    cfg.numAttrs = 2;
    CTCB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, a));
    count_launch();
    return CTCB_OK;
}

// co-resident clusters of the (KI, 8) kernel, the largest of its shared-memory footprints
template <int KI>
static int cluster_max_active() {
    constexpr int CS = KI / 2;
    static int max_clusters = -1;
    if (max_clusters < 0) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(CS, 64, 2);
        cfg.blockDim = dim3(512);
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = CS; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        int n = 0;
        cfg.dynamicSmemBytes = cluster_smem_bytes(KI, 8);
        cudaFuncSetAttribute((sweep_cluster_kernel<KI, 8>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cluster_smem_bytes(KI, 8));
        if (cudaOccupancyMaxActiveClusters(&n, (sweep_cluster_kernel<KI, 8>), &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
        max_clusters = n;
    }
    return max_clusters;
}

// The cluster plan for (H, B, ndir): false where the kernel does not apply (H not 128/256/512, or one wave of clusters
// cannot hold the batch and CTCB_SWEEP_NB does not force a group size)
bool sweep_cluster_plan(int H, int B, int ndir, SweepPlan *p) {
    int max_clusters;
    switch (H) {
        case 128: max_clusters = cluster_max_active<4>(); break;
        case 256: max_clusters = cluster_max_active<8>(); break;
        case 512: max_clusters = cluster_max_active<16>(); break;
        default: return false;
    }
    if (max_clusters < 1) return false;
    // fewest utterances per cluster (= least arithmetic per SM and step) that still fits one wave of clusters
    int nb = 0;
    for (int c = 1; c <= 8; ++c)
        if (ndir * ((B + c - 1) / c) <= max_clusters) { nb = c; break; }
    if (knob(KNOB_SWEEP_NB)) nb = knob(KNOB_SWEEP_NB);     // CTCB_SWEEP_NB=1..8 forces the group size
    if (nb == 0) return false;          // would need a second wave of clusters: the general kernel is faster
    *p = SweepPlan{};
    p->kernel = SWEEP_CLUSTER;
    p->KI = H / 32;
    p->cs = H / 64;
    p->groups = nb;
    p->smem = cluster_smem_bytes(H / 32, nb);
    return true;
}

template <int KI>
static int launch_cluster(const SweepClusterArgs &a, int nb, cudaStream_t st) {
    const int ntiles = (a.B + nb - 1) / nb;
    switch (nb) {
        case 1: return launch_cluster_nb<KI, 1>(a, ntiles, st);
        case 2: return launch_cluster_nb<KI, 2>(a, ntiles, st);
        case 3: return launch_cluster_nb<KI, 3>(a, ntiles, st);
        case 4: return launch_cluster_nb<KI, 4>(a, ntiles, st);
        case 5: return launch_cluster_nb<KI, 5>(a, ntiles, st);
        case 6: return launch_cluster_nb<KI, 6>(a, ntiles, st);
        case 7: return launch_cluster_nb<KI, 7>(a, ntiles, st);
        default: return launch_cluster_nb<KI, 8>(a, ntiles, st);
    }
}

int run_sweep_cluster(const SweepPlan &p, int mode, int T, int B, int H, const int32_t *Tlen, const float *pre,
                      const float *Wf, const float *Wb, float *outF, float *outB, const float *actF, const float *actB,
                      float maxAct, unsigned int *err, cudaStream_t st) {
    SweepClusterArgs a;
    a.mode = mode; a.T = T; a.B = B; a.H = H; a.Tlen = Tlen; a.pre = pre;
    a.W[0] = Wf; a.W[1] = Wb; a.out[0] = outF; a.out[1] = outB; a.act[0] = actF; a.act[1] = actB; a.maxAct = maxAct; a.err = err;
    a.ndir = Wb ? 2 : 1;
    if (!Wb) { a.W[1] = Wf; a.out[1] = outF; a.act[1] = actF; }
    switch (H) {
        case 128: return launch_cluster<4>(a, p.groups, st);
        case 256: return launch_cluster<8>(a, p.groups, st);
        case 512: return launch_cluster<16>(a, p.groups, st);
        default: return set_error(CTCB_EINVAL, "cluster sweep: layerSize %d is not 128, 256 or 512", H);
    }
}

}  // namespace ctcb
