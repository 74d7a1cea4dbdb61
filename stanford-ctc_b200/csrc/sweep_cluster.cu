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
//     cp.async.bulk (shared::cta -> shared::cluster); the copies complete_tx on the DESTINATION's mbarrier,
//     which is the only inter-CTA synchronisation of the step: a CTA starts step s as soon as the CS blocks of
//     step s-1 have landed.  Two state buffers / two barriers alternate;
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
    unsigned long long *mbar = reinterpret_cast<unsigned long long *>(sc_smem + (2 * CS + 32) * BLKF);

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

    const uint32_t bar0 = smem_u32(&mbar[0]), bar1 = smem_u32(&mbar[1]);
    if (tid == 0) {
        mbar_init(bar0, 1);
        mbar_init(bar1, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_arrive_expect_tx(bar0, CS * BLK_BYTES);
        mbar_arrive_expect_tx(bar1, CS * BLK_BYTES);
    }
    cluster_sync_all();

    // epilogue role: thread (eu, ej) = (utterance, unit) for tid < NB*64
    const int eu = tid >> 6, ej = tid & 63;
    const int b = b0 + eu, oj = j0 + ej;
    const bool owner = tid < BLKF;
    const bool valid = owner && (b < B);
    const int Tb = valid ? __ldg(a.Tlen + b) : 0;
    // where this warp's slice of the state sits inside a buffer: source CTA k0/64, offset k0%64
    const int hoff = (k0 >> 6) * BLKF + (k0 & 63);
    bool dead = false;

    for (int s = 0; s < T; ++s) {
        const int t = ascending ? s : T - 1 - s;
        float pre_v = 0.f, act_v = 0.f;
        if (valid) {
            const int64_t o = ((int64_t)t * B + b) * H + oj;
            pre_v = __ldg(a.pre + o);
            if (bptt) act_v = __ldg(act + o);
        }
        float sum = 0.f;
        if (s > 0) {
            const uint32_t bar = (s & 1) ? bar1 : bar0;
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
            __syncthreads();            // the only CTA barrier of the step (red is double-buffered)
            // every warp is past its wait on this step's barrier: arm it for step s + 2
            if (tid == 0 && s + 2 < T) mbar_arrive_expect_tx(bar, CS * BLK_BYTES);
            if (owner) {
                float s0 = 0.f, s1 = 0.f;
#pragma unroll
                for (int w = 0; w < 16; w += 2) { s0 += red[s & 1][w][tid]; s1 += red[s & 1][w + 1][tid]; }
                sum = s0 + s1;
            }
        }
        float v = 0.f;
        if (valid) {
            v = pre_v + sum;
            if (!bptt) v = fminf(fmaxf(v, 0.f), a.maxAct);
            else v = (act_v > 0.f && act_v < a.maxAct) ? v : 0.f;
            if (t >= Tb) v = 0.f;
            out[((int64_t)t * B + b) * H + oj] = v;
        }
        if (owner && s + 1 < T) {
            // hand the new state to every CTA of the cluster (this one included): one remote 4-byte store per
            // peer, each completing 4 bytes on the peer's barrier of step s + 1
            const int nb = (s + 1) & 1;
            const uint32_t dst = smem_u32(&hbuf[nb][rank * BLKF + tid]);
            const uint32_t dbar = nb ? bar1 : bar0;
#pragma unroll
            for (int c = 0; c < CS; ++c) st_async_f32(map_to_cta(dst, (uint32_t)c), v, map_to_cta(dbar, (uint32_t)c));
        }
    }
    cluster_sync_all();
}

static constexpr size_t cluster_smem_bytes(int KI, int NB) {
    return sizeof(float) * (size_t)(2 * (KI / 2) + 32) * (size_t)(NB * 64) + 16;
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
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    CTCB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, a));
    count_launch();
    return CTCB_OK;
}

template <int KI>
static int launch_cluster(const SweepClusterArgs &a, cudaStream_t st, bool *handled) {
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
        if (getenv("CTCB_DEBUG")) fprintf(stderr, "[ctcb] cluster sweep H=%d: cluster=%d CTAs, max active clusters=%d\n", 32 * KI, CS, n);
    }
    *handled = false;
    if (max_clusters < 1) return CTCB_OK;
    static int nb_env = -1;   // CTCB_SWEEP_NB=1..8 forces the group size
    if (nb_env < 0) { const char *e = getenv("CTCB_SWEEP_NB"); nb_env = e ? atoi(e) : 0; }
    // fewest utterances per cluster (= least arithmetic per SM and step) that still fits one wave of clusters
    int nb = 0;
    for (int c = 1; c <= 8; ++c)
        if (a.ndir * ((a.B + c - 1) / c) <= max_clusters) { nb = c; break; }
    if (nb_env >= 1 && nb_env <= 8) nb = nb_env;
    if (nb == 0) return CTCB_OK;          // would need a second wave of clusters: the general kernel is faster
    const int ntiles = (a.B + nb - 1) / nb;
    int rc;
    switch (nb) {
        case 1: rc = launch_cluster_nb<KI, 1>(a, ntiles, st); break;
        case 2: rc = launch_cluster_nb<KI, 2>(a, ntiles, st); break;
        case 3: rc = launch_cluster_nb<KI, 3>(a, ntiles, st); break;
        case 4: rc = launch_cluster_nb<KI, 4>(a, ntiles, st); break;
        case 5: rc = launch_cluster_nb<KI, 5>(a, ntiles, st); break;
        case 6: rc = launch_cluster_nb<KI, 6>(a, ntiles, st); break;
        case 7: rc = launch_cluster_nb<KI, 7>(a, ntiles, st); break;
        default: rc = launch_cluster_nb<KI, 8>(a, ntiles, st); break;
    }
    if (rc == CTCB_OK) *handled = true;
    return rc;
}

int run_sweep_cluster(int mode, int T, int B, int H, const int32_t *Tlen, const float *pre, const float *Wf,
                      const float *Wb, float *outF, float *outB, const float *actF, const float *actB, float maxAct,
                      unsigned int *err, cudaStream_t st, bool *handled) {
    *handled = false;
    if (H != 128 && H != 256 && H != 512) return CTCB_OK;
    SweepClusterArgs a;
    a.mode = mode; a.T = T; a.B = B; a.H = H; a.Tlen = Tlen; a.pre = pre;
    a.W[0] = Wf; a.W[1] = Wb; a.out[0] = outF; a.out[1] = outB; a.act[0] = actF; a.act[1] = actB; a.maxAct = maxAct; a.err = err;
    a.ndir = Wb ? 2 : 1;
    if (!Wb) { a.W[1] = Wf; a.out[1] = outF; a.act[1] = actF; }
    switch (H / 32) {
        case 4: return launch_cluster<4>(a, st, handled);
        case 8: return launch_cluster<8>(a, st, handled);
        case 16: return launch_cluster<16>(a, st, handled);
        default: return CTCB_OK;
    }
}

}  // namespace ctcb
