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
#include "common.cuh"
#include <stdlib.h>

namespace ctcb {

constexpr int SW_THREADS = 256;
constexpr int SW_ROWS = 32;   // output units per CTA (4 per warp)
constexpr int SW_NB = 8;      // utterances per inner tile

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
    unsigned int *counters; // [2 * parts], zeroed before launch
};

__device__ __forceinline__ void domain_barrier(unsigned int *ctr, unsigned int target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(ctr, 1u);
        unsigned int v;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
        } while (v < target);
    }
    __syncthreads();
}

// KI > 0: H == 32*KI and the weights live in registers.  KI == 0: any H, weights re-read through L1/L2.
template <int KI>
__global__ void __launch_bounds__(SW_THREADS, 1) sweep_kernel(SweepArgs a) {
    extern __shared__ __align__(16) float hs[];   // [SW_NB][Hp]
    const int H = a.H, B = a.B, T = a.T;
    const int Hp = (H + 3) / 4 * 4 + 4;
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
    // utterance range of this partition, in tiles of SW_NB
    const int ntiles = (B + SW_NB - 1) / SW_NB;
    const int tiles_per_part = (ntiles + a.parts - 1) / a.parts;
    const int tile_beg = blockIdx.y * tiles_per_part;
    const int tile_end = min(ntiles, tile_beg + tiles_per_part);
    unsigned int *ctr = a.counters + (dir * a.parts + blockIdx.y);
    const unsigned int nslices = gridDim.x;

    // lane -> (row r, utterance b) of the value it ends up owning after the transposing reduction
    const int orow = lane >> 3, ob = lane & 7;
    const int oj = j0 + orow;

    for (int s = 0; s < T; ++s) {
        const int t = ascending ? s : T - 1 - s;
        const int tprev = ascending ? t - 1 : t + 1;
        for (int tile = tile_beg; tile < tile_end; ++tile) {
            const int b0 = tile * SW_NB;
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
                // previous state of this tile's utterances: [SW_NB][H] from L2 -> shared
                const float *src = out + ((int64_t)tprev * B + b0) * H;
                const int nb = min(SW_NB, B - b0);
                if ((H & 3) == 0) {
                    const int h4 = H >> 2;
                    for (int idx = threadIdx.x; idx < nb * h4; idx += SW_THREADS) {
                        const int bb = idx / h4, k4 = idx - bb * h4;
                        const float4 v = __ldcg(reinterpret_cast<const float4 *>(src + (int64_t)bb * H) + k4);
                        *reinterpret_cast<float4 *>(hs + bb * Hp + 4 * k4) = v;
                    }
                } else {
                    for (int idx = threadIdx.x; idx < nb * H; idx += SW_THREADS) {
                        const int bb = idx / H, k = idx - bb * H;
                        hs[bb * Hp + k] = __ldcg(src + (int64_t)bb * H + k);
                    }
                }
                for (int idx = threadIdx.x + nb * Hp; idx < SW_NB * Hp; idx += SW_THREADS) hs[idx] = 0.f;
                __syncthreads();
                if (KI > 0) {
#pragma unroll
                    for (int i = 0; i < KI; ++i) {
                        float hv[SW_NB];
#pragma unroll
                        for (int bb = 0; bb < SW_NB; ++bb) hv[bb] = hs[bb * Hp + lane + 32 * i];
#pragma unroll
                        for (int r = 0; r < 4; ++r)
#pragma unroll
                            for (int bb = 0; bb < SW_NB; ++bb)
                                acc[r * 8 + bb] = fmaf(wreg[r][i], hv[bb], acc[r * 8 + bb]);
                    }
                } else {
                    for (int k = lane; k < H; k += 32) {
                        float hv[SW_NB], wv[4];
#pragma unroll
                        for (int bb = 0; bb < SW_NB; ++bb) hv[bb] = hs[bb * Hp + k];
#pragma unroll
                        for (int r = 0; r < 4; ++r) {
                            const int j = j0 + r;
                            wv[r] = (j < H) ? (bptt ? __ldg(W + (int64_t)k * H + j) : __ldg(W + (int64_t)j * H + k)) : 0.f;
                        }
#pragma unroll
                        for (int r = 0; r < 4; ++r)
#pragma unroll
                            for (int bb = 0; bb < SW_NB; ++bb)
                                acc[r * 8 + bb] = fmaf(wv[r], hv[bb], acc[r * 8 + bb]);
                    }
                }
                // transposing butterfly: lane l ends with sum over lanes of acc[l]
#pragma unroll
                for (int off = 16, n = 32; off >= 1; off >>= 1, n >>= 1) {
                    const bool up = (lane & off) != 0;
#pragma unroll
                    for (int i = 0; i < n / 2; ++i) {
                        const float send = up ? acc[i] : acc[i + n / 2];
                        const float keep = up ? acc[i + n / 2] : acc[i];
                        acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                    }
                }
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
        if (s + 1 < T) domain_barrier(ctr, nslices * (unsigned int)(s + 1));
    }
}

__global__ void add2_kernel(const float *__restrict__ x, const float *__restrict__ y, float *__restrict__ z, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) z[i] = x[i] + y[i];
}

template <int KI>
static int launch_sweep(SweepArgs &a, int slices, size_t smem, cudaStream_t st) {
    int dev = 0, per_sm = 0;
    CTCB_CUDA_CHECK(cudaGetDevice(&dev));
    CTCB_CUDA_CHECK(cudaFuncSetAttribute(sweep_kernel<KI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CTCB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sweep_kernel<KI>, SW_THREADS, smem));
    const int capacity = per_sm * num_sms();
    if (a.ndir * slices > capacity)
        return set_error(CTCB_EINVAL, "recurrent sweep: layerSize %d needs %d co-resident CTAs, device holds %d",
                         a.H, a.ndir * slices, capacity);
    const int ntiles = (a.B + SW_NB - 1) / SW_NB;
    int parts = capacity / (a.ndir * slices);
    if (parts > ntiles) parts = ntiles;
    if (parts > 500) parts = 500;   // counters region holds 1024 words
    if (parts < 1) parts = 1;
    a.parts = parts;
    a.counters += 16;     // words [0..15] are reserved for error flags, which the CALLER clears (once per step)
    CTCB_CUDA_CHECK(cudaMemsetAsync(a.counters, 0, sizeof(unsigned int) * (a.ndir * parts), st));
    dim3 grid(slices, parts, a.ndir);
    void *params[] = {&a};
    CTCB_CUDA_CHECK(cudaLaunchCooperativeKernel((void *)sweep_kernel<KI>, grid, dim3(SW_THREADS), params, smem, st));
    count_launch();
    return CTCB_OK;
}

int run_sweep_cluster(int mode, int T, int B, int H, const int32_t *Tlen, const float *pre, const float *Wf,
                      const float *Wb, float *outF, float *outB, const float *actF, const float *actB, float maxAct,
                      unsigned int *err, cudaStream_t st, bool *handled);
int run_sweep_tc(int mode, int T, int B, int H, const int32_t *Tlen, const float *pre, const float *Wf, const float *Wb,
                 float *outF, float *outB, const float *actF, const float *actB, float maxAct, unsigned int *counters,
                 void *ws, size_t ws_bytes, cudaStream_t st, bool *handled);

// counters: 4096 bytes of device scratch (word 0 = error flag, cleared by the caller); ws: optional further scratch
// (sweep_tc_workspace_bytes(H)) that lets the tensor-core kernel run the BPTT mode as well
int run_sweep(int mode, int T, int B, int H, const int32_t *Tlen, const float *pre, const float *Wf,
              const float *Wb, float *outF, float *outB, const float *actF, const float *actB, float maxAct,
              unsigned int *counters, void *ws, size_t ws_bytes, cudaStream_t st) {
    {   // tensor-core path (H >= 1024)
        bool handled = false;
        const int rc = run_sweep_tc(mode, T, B, H, Tlen, pre, Wf, Wb, outF, outB, actF, actB, maxAct, counters, ws, ws_bytes, st, &handled);
        if (rc != CTCB_OK) return rc;
        if (handled) return CTCB_OK;
    }
    SweepArgs a;
    a.mode = mode; a.T = T; a.B = B; a.H = H; a.Tlen = Tlen; a.pre = pre;
    a.W[0] = Wf; a.W[1] = Wb; a.out[0] = outF; a.out[1] = outB; a.act[0] = actF; a.act[1] = actB;
    a.maxAct = maxAct; a.counters = counters; a.parts = 1;
    a.ndir = Wb ? 2 : 1;
    if (!Wb) { a.W[1] = Wf; a.out[1] = outF; a.act[1] = actF; }   // never dereferenced: gridDim.z == 1
    {   // cluster/DSMEM fast path (H = 128, 256, 512); CTCB_SWEEP=barrier forces the general kernel
        static int force_barrier = -1;
        if (force_barrier < 0) {
            const char *e = getenv("CTCB_SWEEP");
            force_barrier = (e && e[0] == 'b') ? 1 : 0;
        }
        if (!force_barrier) {
            bool handled = false;
            const int rc = run_sweep_cluster(mode, T, B, H, Tlen, pre, Wf, Wb, outF, outB, actF, actB, maxAct, counters, st, &handled);
            if (rc == CTCB_OK && handled) return CTCB_OK;
            if (rc != CTCB_OK) cudaGetLastError();   // cluster launch refused: fall through to the general kernel
        }
    }
    const int slices = (H + SW_ROWS - 1) / SW_ROWS;
    const int Hp = (H + 3) / 4 * 4 + 4;
    const size_t smem = (size_t)SW_NB * Hp * sizeof(float);
    if (H % 32 == 0) {
        switch (H / 32) {
            case 4: return launch_sweep<4>(a, slices, smem, st);
            case 8: return launch_sweep<8>(a, slices, smem, st);
            case 16: return launch_sweep<16>(a, slices, smem, st);
            case 32: return launch_sweep<32>(a, slices, smem, st);
            default: break;
        }
    }
    return launch_sweep<0>(a, slices, smem, st);
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
