// Microbenchmark for the open question of the cluster sweep (DESIGN.md section 6): what does a warp-uniform
// (broadcast) LDS.128, a full-width LDS.128 and a SHFL cost per SM when 16 warps issue them back to back, alone
// and interleaved with the FFMA pairs of the sweep?  Prints cycles per instruction per SM sub-partition.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o lsu_rate lsu_rate.cu ; run: ./lsu_rate
#include <cstdio>
#include <cuda_runtime.h>

// a pair of output units times one scalar, as sweep_cluster.cu computes it: two FFMA
__device__ __forceinline__ void ffma2(unsigned long long &d, unsigned long long a, float h) {
    float dl, dh, al, ah;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(dl), "=f"(dh) : "l"(d));
    asm("mov.b64 {%0, %1}, %2;" : "=f"(al), "=f"(ah) : "l"(a));
    dl = fmaf(al, h, dl);
    dh = fmaf(ah, h, dh);
    asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(dl), "f"(dh));
}

// MODE 0: broadcast LDS.128 (all lanes one address)   1: full-width LDS.128 (lane-consecutive 16 B)
// MODE 2: SHFL.BFLY                                   3: broadcast LDS.128 + 4 FFMA pairs each (the sweep's inner loop)
template <int MODE>
__global__ void k(float *out, long long *cycles, int iters) {
    __shared__ __align__(16) float sm[32 * 4 * 16 + 64];
    for (int i = threadIdx.x; i < 32 * 4 * 16 + 64; i += blockDim.x) sm[i] = 1.0f + i * 1e-6f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    float acc = 0.f;
    unsigned long long d[4] = {0ull, 0ull, 0ull, 0ull};
    const unsigned long long w = 0x3f8000003f000000ull;
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            if (MODE == 0 || MODE == 3) {
                const float4 v = *reinterpret_cast<const float4 *>(&sm[4 * ((q + it) & 15)]);
                if (MODE == 0) acc += v.x + v.y + v.z + v.w;
                else { ffma2(d[0], w, v.x); ffma2(d[1], w, v.y); ffma2(d[2], w, v.z); ffma2(d[3], w, v.w); }
            } else if (MODE == 1) {
                const float4 v = *reinterpret_cast<const float4 *>(&sm[4 * (lane + 32 * ((q + it) & 15))]);
                acc += v.x + v.y + v.z + v.w;
            } else {
                acc += __shfl_xor_sync(0xffffffffu, acc + q, 1 + (q & 15));
            }
        }
    }
    const long long t1 = clock64();
    for (int i = 0; i < 4; ++i) acc += (float)(d[i] & 0xffff);
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

static int nsm() {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
    return n;
}

template <int MODE>
static void run(const char *name, float *out, long long *cyc) {
    const int iters = 500;
    for (int warps : {4, 16}) {
        long long h[1];
        k<MODE><<<nsm(), warps * 32>>>(out, cyc, iters);
        cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
        const double per_sm = (double)h[0] / (iters * 16.0 * warps);          // cycles per instruction, whole SM
        printf("%-34s %2d warps/SM: %.2f cycles per warp instruction per SM (%.2f per sub-partition)\n", name, warps,
               per_sm, per_sm * 4);
    }
}

int main() {
    float *out; long long *cyc;
    cudaMalloc(&out, nsm() * 512 * sizeof(float));
    cudaMalloc(&cyc, nsm() * sizeof(long long));
    run<0>("broadcast LDS.128", out, cyc);
    run<1>("full-width LDS.128", out, cyc);
    run<2>("SHFL.BFLY", out, cyc);
    run<3>("broadcast LDS.128 + 4 FFMA pairs", out, cyc);
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
