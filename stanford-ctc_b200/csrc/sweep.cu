// sweep.cu -- the bi-directional time recurrences of the temporal layer as ONE persistent kernel.
//
// Replaces the 4(T-1) cudamat launches per utterance of the reference's hot loops
//   forward : For[:,t]  = clip(pre[:,t] + Wtf.For[:,t-1], 0, 20),  Back mirrored
//             (ctc_fast/nnets/brnnet.py:144-152: mvdot_col_slice + minmax)
//   BPTT    : dFor[:,t] = within(For[:,t]) * (d[:,t] + Wtf^T.dFor[:,t+1]),  dBack mirrored
//             (brnnet.py:208-224: mvdot_col_slice on W.T + mult_slice)
// with a batch of utterances as the second matrix dimension.
//
// Three kernels share this design point (run_sweep below picks one):
//   * sweep_tc.cu (layerSize >= 1024, round 2): the step as a wgmma tensor-core contraction spread over the device,
//     split-K partials reduced through DSMEM, one counter barrier per step.
//   * sweep_cluster.cu (H = 128/256/512): one thread-block cluster per (direction, 8 utterances); the
//     hidden state is exchanged CTA-to-CTA through distributed shared memory with bulk async copies
//     that complete on the consumer's mbarrier -- no global-memory round trip on the serial chain.
//   * this file (any H): the general fallback below, exchanging through L2 with a counter barrier.
//
// Design: the H x H recurrent matrix never leaves the register file.  A CTA of 8 warps owns
// 32 output units; lane l of warp w keeps W[j][l + 32 i] for its 4 rows j in registers for the
// whole sweep (H/32 * 4 registers), so a time step only moves the previous hidden state
// (8 utterances x H floats, read from L2 into shared memory) and the 32 x 8 new outputs.  Both
// directions run concurrently in the same launch (blockIdx.z).  CTAs that share a (direction,
// utterance partition) synchronise once per time step through a monotonically increasing counter
// in global memory (cooperative launch guarantees co-residency); the hidden state itself is
// exchanged through the output array in L2 (ld.global.cg), which has to be written anyway.
//
// Data layout: time-major [T][B][H] fp32, so one time step of all utterances is contiguous.
//
// From coop_sweep.cuh, which the LSTM sweep (sweep_lstm.cu) shares: the block and tile sizes, the state-tile load, the
// transposing butterfly, the partition's tiles, the bounded step barrier (a timeout sets the error flag to 1), and on
// the host the partition planner, the KI dispatch and the cooperative launch.
#include "coop_sweep.cuh"
#include <stdlib.h>

namespace ctcb {

constexpr int SW_ROWS = 32;   // output units per CTA (4 per warp)

struct SweepArgs {
    int mode;               // 0: forward recurrences, 1: BPTT
    int T, B, H;
    const int32_t *Tlen;    // [B]
    const float *pre;       // mode 0: pre-activations [T][B][H]; mode 1: incoming deltas
    const float *W[2];      // Wtf, Wtb  (H x H, row-major out x in)
    float *out[2];          // mode 0: For, Back; mode 1: dFor, dBack
    const float *act[2];    // mode 1: For, Back (for the within(0,maxAct) masks)
    float maxAct;
    int parts;              // utterance partitions (gridDim.y)
    int ndir;               // 2: forward and backward direction (gridDim.z); 1: forward in time only
    unsigned int *err;      // word 0 of the scratch: the error flag, cleared by the caller
    unsigned int *counters; // [ndir * parts], zeroed before launch
};

// KI > 0: H == 32*KI and the weights live in registers.  KI == 0: any H, weights re-read through L1/L2, at three CTAs
// per SM (at most 80 registers), which sets how wide a layer the device holds co-resident.
template <int KI>
__global__ void __launch_bounds__(COOP_THREADS, KI > 0 ? 1 : 3) sweep_kernel(SweepArgs a) {
    extern __shared__ __align__(16) float hs[];   // [COOP_NB][Hp]
    const int H = a.H, B = a.B, T = a.T;
    const int Hp = coop_hp(H);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int dir = blockIdx.z;
    const int j0 = blockIdx.x * SW_ROWS + warp * 4;
    const float *W = a.W[dir];
    float *out = a.out[dir];
    const bool bptt = (a.mode == 1);
    // time runs forward for (forward-mode, dir 0) and (BPTT, dir 1)
    const bool ascending = (dir == 0) != bptt;
    // contraction: forward uses W (row j), BPTT uses W^T (column j)
    float wreg[4][KI > 0 ? KI : 1];
    if (KI > 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int i = 0; i < KI; ++i) {
                const int j = j0 + r, k = lane + 32 * i;
                wreg[r][i] = (j < H) ? (bptt ? W[(int64_t)k * H + j] : W[(int64_t)j * H + k]) : 0.f;
            }
    }
    int tile_beg, tile_end;
    coop_tile_range(B, a.parts, tile_beg, tile_end);
    unsigned int *ctr = a.counters + (dir * a.parts + blockIdx.y);
    const unsigned int nslices = gridDim.x;
    bool dead = false;

    // lane -> (row r, utterance b) of the value it ends up owning after the transposing reduction
    const int orow = lane >> 3, ob = lane & 7;
    const int oj = j0 + orow;

    for (int s = 0; s < T; ++s) {
        const int t = ascending ? s : T - 1 - s;
        const int tprev = ascending ? t - 1 : t + 1;
        for (int tile = tile_beg; tile < tile_end; ++tile) {
            const int b0 = tile * COOP_NB;
            const int b = b0 + ob;
            // issue the epilogue operands early: they do not depend on the recurrence
            float pre_v = 0.f, act_v = 0.f;
            int Tb = 0;
            const bool valid = (oj < H) && (b < B);
            if (valid) {
                const int64_t o = ((int64_t)t * B + b) * H + oj;
                pre_v = __ldg(a.pre + o);
                if (bptt) act_v = __ldg(a.act[dir] + o);
                Tb = __ldg(a.Tlen + b);
            }
            float acc[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = 0.f;
            if (s > 0) {
                // previous state of this tile's utterances from L2
                coop_load_state(hs, Hp, out + ((int64_t)tprev * B + b0) * H, H, min(COOP_NB, B - b0), H);
                __syncthreads();
                if (KI > 0) {
#pragma unroll
                    for (int i = 0; i < KI; ++i) {
                        float hv[COOP_NB];
#pragma unroll
                        for (int bb = 0; bb < COOP_NB; ++bb) hv[bb] = hs[bb * Hp + lane + 32 * i];
#pragma unroll
                        for (int r = 0; r < 4; ++r)
#pragma unroll
                            for (int bb = 0; bb < COOP_NB; ++bb)
                                acc[r * 8 + bb] = fmaf(wreg[r][i], hv[bb], acc[r * 8 + bb]);
                    }
                } else {
                    for (int k = lane; k < H; k += 32) {
                        float hv[COOP_NB], wv[4];
#pragma unroll
                        for (int bb = 0; bb < COOP_NB; ++bb) hv[bb] = hs[bb * Hp + k];
#pragma unroll
                        for (int r = 0; r < 4; ++r) {
                            const int j = j0 + r;
                            wv[r] = (j < H) ? (bptt ? __ldg(W + (int64_t)k * H + j) : __ldg(W + (int64_t)j * H + k)) : 0.f;
                        }
#pragma unroll
                        for (int r = 0; r < 4; ++r)
#pragma unroll
                            for (int bb = 0; bb < COOP_NB; ++bb)
                                acc[r * 8 + bb] = fmaf(wv[r], hv[bb], acc[r * 8 + bb]);
                    }
                }
                coop_butterfly(acc, lane);
                __syncthreads();   // hs is reused by the next tile
            }
            if (valid) {
                float v = pre_v + acc[0];
                if (!bptt) {
                    v = fminf(fmaxf(v, 0.f), a.maxAct);          // minmax(0, maxAct)
                    if (t >= Tb) v = 0.f;                        // beyond the utterance: zero state
                } else {
                    v = (act_v > 0.f && act_v < a.maxAct) ? v : 0.f;   // within(0, maxAct)
                    if (t >= Tb) v = 0.f;
                }
                out[((int64_t)t * B + b) * H + oj] = v;
            }
        }
        if (s + 1 < T) coop_barrier(ctr, nslices * (unsigned int)(s + 1), a.err, 1u, dead);
    }
}

__global__ void add2_kernel(const float *__restrict__ x, const float *__restrict__ y, float *__restrict__ z, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) z[i] = x[i] + y[i];
}

bool sweep_tc_plan(int H, int B, int ndir, SweepPlan *p);
bool sweep_cluster_plan(int H, int B, int ndir, SweepPlan *p);
int run_sweep_cluster(const SweepPlan &p, int mode, int T, int B, int H, const int32_t *Tlen, const float *pre,
                      const float *Wf, const float *Wb, float *outF, float *outB, const float *actF, const float *actB,
                      float maxAct, unsigned int *err, cudaStream_t st);
int run_sweep_tc(const SweepPlan &p, int mode, int T, int B, int H, const int32_t *Tlen, const float *pre, const float *Wf,
                 const float *Wb, float *outF, float *outB, const float *actF, const float *actB, float maxAct,
                 unsigned int *counters, void *ws, size_t ws_bytes, cudaStream_t st);

// The one place that decides which kernel runs a sweep of (H, B, ndir): the tensor-core kernel where it applies
// (H >= 1024, CTCB_SWEEP_TC), else the cluster kernel (H = 128/256/512; CTCB_SWEEP=barrier or reread skips it), else the
// generic kernel, whose CTAs must all be co-resident.  CTCB_SWEEP=reread takes the generic kernel's KI = 0 at any H;
// CTCB_SWEEP_PARTS forces its partition count.  A width whose shared memory or CTAs the device cannot hold, or a forced
// count it cannot hold co-resident, is refused here, before any launch.
int select_sweep(int H, int B, int ndir, SweepPlan *p) {
    if (H <= 0 || B <= 0 || (ndir != 1 && ndir != 2))
        return set_error(CTCB_EINVAL, "recurrent sweep: bad sizes (H=%d, B=%d, ndir=%d)", H, B, ndir);
    if (sweep_tc_plan(H, B, ndir, p)) return CTCB_OK;
    if (!knob(KNOB_SWEEP) && sweep_cluster_plan(H, B, ndir, p)) return CTCB_OK;
    *p = SweepPlan{};
    p->kernel = SWEEP_GENERIC;
    const bool reg = (H == 128 || H == 256 || H == 512 || H == 1024) && knob(KNOB_SWEEP) != 2;
    p->KI = reg ? H / 32 : 0;
    p->smem = coop_smem(H);
    if (p->smem > max_smem_optin())
        return set_error(CTCB_EINVAL, "recurrent sweep: layerSize %d needs %zu bytes of shared memory per CTA, device "
                         "allows %zu", H, p->smem, max_smem_optin());
    const int rc = with_ki<4, 8, 16, 32>(p->KI, [&](auto ki) {
        return coop_occupancy(sweep_kernel<decltype(ki)::value>, p->smem, &p->per_sm);
    });
    if (rc != CTCB_OK) return rc;
    return coop_parts("recurrent sweep", H, p->per_sm, ndir, (H + SW_ROWS - 1) / SW_ROWS, B, knob(KNOB_SWEEP_PARTS),
                      "CTCB_SWEEP_PARTS", &p->groups);
}

// ctcb_brnn_create's check that the device holds the ReLU sweep of a config at its largest batch (every plan that holds
// maxB holds a smaller batch)
int sweep_check(int H, int B, int ndir) {
    if (no_device()) return CTCB_OK;
    SweepPlan p;
    return select_sweep(H, B, ndir, &p);
}

// counters: 4096 bytes of device scratch (word 0 = error flag, cleared by the caller); ws: optional further scratch
// (sweep_tc_workspace_bytes(H)) that lets the tensor-core kernel run the BPTT mode as well
int run_sweep(int mode, int T, int B, int H, const int32_t *Tlen, const float *pre, const float *Wf,
              const float *Wb, float *outF, float *outB, const float *actF, const float *actB, float maxAct,
              unsigned int *counters, void *ws, size_t ws_bytes, cudaStream_t st) {
    SweepPlan p;
    const int rc = select_sweep(H, B, Wb ? 2 : 1, &p);
    if (rc != CTCB_OK) return rc;
    if (p.kernel == SWEEP_TC)
        return run_sweep_tc(p, mode, T, B, H, Tlen, pre, Wf, Wb, outF, outB, actF, actB, maxAct, counters, ws, ws_bytes, st);
    if (p.kernel == SWEEP_CLUSTER)
        return run_sweep_cluster(p, mode, T, B, H, Tlen, pre, Wf, Wb, outF, outB, actF, actB, maxAct, counters, st);
    SweepArgs a;
    a.mode = mode; a.T = T; a.B = B; a.H = H; a.Tlen = Tlen; a.pre = pre;
    a.W[0] = Wf; a.W[1] = Wb; a.out[0] = outF; a.out[1] = outB; a.act[0] = actF; a.act[1] = actB;
    a.maxAct = maxAct;
    a.ndir = Wb ? 2 : 1;
    if (!Wb) { a.W[1] = Wf; a.out[1] = outF; a.act[1] = actF; }   // never dereferenced: gridDim.z == 1
    return with_ki<4, 8, 16, 32>(p.KI, [&](auto ki) {
        return coop_launch(sweep_kernel<decltype(ki)::value>, a, counters, (H + SW_ROWS - 1) / SW_ROWS, p.groups, p.smem,
                           st);
    });
}

int run_add2(const float *x, const float *y, float *z, int64_t n, cudaStream_t st) {
    int blocks = (int)((n + 1023) / 1024);
    if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
    if (blocks < 1) blocks = 1;
    add2_kernel<<<blocks, 256, 0, st>>>(x, y, z, n);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb

extern "C" int ctcb_debug_sweep_plan(int H, int B, int ndir, int32_t *out) {
    if (!out) return ctcb::set_error(CTCB_EINVAL, "ctcb_debug_sweep_plan: null output");
    ctcb::SweepPlan p;
    const int rc = ctcb::select_sweep(H, B, ndir, &p);
    if (rc != CTCB_OK) return rc;
    const int32_t v[8] = {p.kernel, p.KI, p.cs, p.groups, p.np, p.stages, p.partial_own,
                          p.kernel == ctcb::SWEEP_GENERIC ? p.per_sm : 0};
    for (int i = 0; i < 8; ++i) out[i] = v[i];
    return CTCB_OK;
}

extern "C" int ctcb_debug_sweep_plan_tf32(int H, int B, int ndir, int32_t *out) {
    ctcb::Tf32Scope tf32(1);
    return ctcb_debug_sweep_plan(H, B, ndir, out);
}

extern "C" int ctcb_sweep_uses_tensor_cores(int H, int B) {
    ctcb::SweepPlan p;
    return (ctcb::select_sweep(H, B, 2, &p) == CTCB_OK && p.kernel == ctcb::SWEEP_TC) ? 1 : 0;
}
