// coop_sweep.cuh -- the scaffold of the two cooperative recurrent sweeps, sweep_kernel<KI> (sweep.cu, clipped ReLU)
// and lstm_sweep_kernel<KI, PEEP> (sweep_lstm.cu).
//
// Both are persistent kernels of COOP_THREADS threads, launched cooperatively on a (slices, parts, ndir) grid, and so
// co-resident across the device.  A CTA walks the COOP_NB-utterance tiles of its partition; for each it loads the
// previous step's state of the tile from L2 into a [COOP_NB][coop_hp(H)] shared tile, accumulates 32 values per lane
// and sums them over the warp with one transposing butterfly.  The CTAs of one (direction, partition) meet once per time
// step at a counter barrier in global memory whose wait is bounded.  How many rows a CTA owns, the arithmetic and the
// stores are each kernel's own and stay in its file.
#pragma once
#include "common.cuh"
#include <type_traits>

namespace ctcb {

constexpr int COOP_THREADS = 256;   // 8 warps per CTA
constexpr int COOP_NB = 8;          // utterances per tile

// The row pitch, in floats, of the shared state tile: 16-byte rows, and 4 floats of padding against bank conflicts
__host__ __device__ constexpr int coop_hp(int H) { return (H + 3) / 4 * 4 + 4; }
__host__ __device__ constexpr int coop_tiles(int B) { return (B + COOP_NB - 1) / COOP_NB; }
inline size_t coop_smem(int H) { return (size_t)COOP_NB * coop_hp(H) * sizeof(float); }

// The per-step barrier of the CTAs of one (direction, partition).  A wait longer than ~0.5 s sets *err to code and
// gives up waiting for the rest of the sweep: the results are invalid, but the sweep ends.
__device__ __forceinline__ void coop_barrier(unsigned int *ctr, unsigned int target, unsigned int *err, unsigned int code,
                                             bool &dead) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(ctr, 1u);
        if (!dead) {
            const long long t0 = clock64();
            while (true) {
                unsigned int v;
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
                if (v >= target) break;
                if (clock64() - t0 > 1000000000LL) {
                    dead = true;
                    atomicExch(err, code);
                    break;
                }
            }
        }
    }
    __syncthreads();
}

// [COOP_NB][Hp] <- nb rows of H floats at src, src + pitch, ...; the rows beyond nb are zeroed
__device__ __forceinline__ void coop_load_state(float *hs, int Hp, const float *src, int64_t pitch, int nb, int H) {
    if ((H & 3) == 0 && (pitch & 3) == 0 && (((uintptr_t)src) & 15) == 0) {
        const int h4 = H >> 2;
        for (int idx = threadIdx.x; idx < nb * h4; idx += COOP_THREADS) {
            const int bb = idx / h4, k4 = idx - bb * h4;
            const float4 v = __ldcg(reinterpret_cast<const float4 *>(src + bb * pitch) + k4);
            *reinterpret_cast<float4 *>(hs + bb * Hp + 4 * k4) = v;
        }
    } else {
        for (int idx = threadIdx.x; idx < nb * H; idx += COOP_THREADS) {
            const int bb = idx / H, k = idx - bb * H;
            hs[bb * Hp + k] = __ldcg(src + bb * pitch + k);
        }
    }
    for (int idx = threadIdx.x + nb * Hp; idx < COOP_NB * Hp; idx += COOP_THREADS) hs[idx] = 0.f;
}

// Transposing butterfly: lane l ends with the sum over the warp's lanes of acc[l], in acc[0]
__device__ __forceinline__ void coop_butterfly(float (&acc)[32], int lane) {
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
}

// The tiles [beg, end) of partition blockIdx.y: the batch's tiles in parts equal runs, the last one shorter or empty
__device__ __forceinline__ void coop_tile_range(int B, int parts, int &beg, int &end) {
    const int ntiles = coop_tiles(B), per_part = (ntiles + parts - 1) / parts;
    beg = blockIdx.y * per_part;
    end = min(ntiles, beg + per_part);
}

// ---- host ----------------------------------------------------------------------------------------------------------

// ctcb_brnn_create checks that the device holds the sweep of a config; without a device there is nothing to check
// against, and the launch checks again
inline bool no_device() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        (void)cudaGetLastError();
        return true;
    }
    return false;
}

// Calls f(std::integral_constant<int, KI>()) for the KI among KIS, else for KI = 0 (the weights re-read): the one place
// a plan's KI picks a kernel instantiation
template <int... KIS, class F>
int with_ki(int KI, F &&f) {
    int rc = CTCB_OK;
    const bool found = ((KI == KIS ? (rc = f(std::integral_constant<int, KIS>()), true) : false) || ...);
    return found ? rc : f(std::integral_constant<int, 0>());
}

// CTAs of kernel one SM holds with this much dynamic shared memory (at most max_smem_optin())
template <class Args>
int coop_occupancy(void (*kernel)(Args), size_t smem, int *per_sm) {
    CTCB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CTCB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, kernel, COOP_THREADS, smem));
    return CTCB_OK;
}

// The utterance partitions of a sweep of ndir * slices CTAs per partition whose kernel one SM holds per_sm of: as many
// as the device holds co-resident, or the count `forced` that the knob knob_name sets, clamped to the batch's tiles, to
// COOP_SWEEP_MAX_PARTS and to at least 1.  A layer, or a forced count, whose CTAs the device cannot hold at once is
// refused here, before any launch.  sweep names the kernel in the error text.
inline int coop_parts(const char *sweep, int H, int per_sm, int ndir, int slices, int B, int forced,
                      const char *knob_name, int *parts) {
    const int capacity = per_sm * num_sms();
    if (ndir * slices > capacity)
        return set_error(CTCB_EINVAL, "%s: layerSize %d needs %d co-resident CTAs, device holds %d", sweep, H,
                         ndir * slices, capacity);
    int n = capacity / (ndir * slices);
    if (forced) {
        if (forced > n)
            return set_error(CTCB_EINVAL, "%s: %s=%d needs %d co-resident CTAs, device holds %d", sweep, knob_name,
                             forced, forced * ndir * slices, capacity);
        n = forced;
    }
    if (n > coop_tiles(B)) n = coop_tiles(B);
    if (n > COOP_SWEEP_MAX_PARTS) n = COOP_SWEEP_MAX_PARTS;
    *parts = n < 1 ? 1 : n;
    return CTCB_OK;
}

// Launches kernel on a (slices, parts, a.ndir) grid with its counters zeroed.  scratch: words 0..15 the error flags
// (word 0 is a.err, which the caller clears), then the [a.ndir][parts] barrier counters.
template <class Args>
int coop_launch(void (*kernel)(Args), Args &a, unsigned int *scratch, int slices, int parts, size_t smem,
                cudaStream_t st) {
    a.err = scratch;
    a.counters = scratch + 16;
    a.parts = parts;
    CTCB_CUDA_CHECK(cudaMemsetAsync(a.counters, 0, sizeof(unsigned int) * (a.ndir * parts), st));
    void *params[] = {&a};
    CTCB_CUDA_CHECK(cudaLaunchCooperativeKernel((void *)kernel, dim3(slices, parts, a.ndir), dim3(COOP_THREADS), params,
                                                smem, st));
    count_launch();
    return CTCB_OK;
}

}  // namespace ctcb
