// Microbenchmark: issue rate of the warp-level mma.sync.m16n8k8 TF32 path and of FFMA on sm_90a.
// One CTA of W warps per SM; each warp runs ITER iterations of NACC independent accumulator chains.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o mma_rate mma_rate.cu ; run: ./mma_rate
#include <cstdio>
#include <cuda_runtime.h>

template <int NACC>
__global__ void mma_kernel(float *out, long long *cycles, int iters) {
    float d[NACC][4];
    unsigned a[4], b[2];
    for (int i = 0; i < 4; ++i) a[i] = __float_as_uint(1.0f + threadIdx.x * 1e-3f + i);
    for (int i = 0; i < 2; ++i) b[i] = __float_as_uint(0.5f + threadIdx.x * 1e-3f + i);
    for (int n = 0; n < NACC; ++n) for (int i = 0; i < 4; ++i) d[n][i] = 0.f;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int n = 0; n < NACC; ++n)
            asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(d[n][0]), "+f"(d[n][1]), "+f"(d[n][2]), "+f"(d[n][3])
                         : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
    const long long t1 = clock64();
    float s = 0.f;
    for (int n = 0; n < NACC; ++n) for (int i = 0; i < 4; ++i) s += d[n][i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int NACC>
__global__ void ffma_kernel(float *out, long long *cycles, int iters) {
    float d[NACC], a[NACC];
    float h = 0.5f + threadIdx.x * 1e-3f;
    for (int n = 0; n < NACC; ++n) { d[n] = 0.f; a[n] = 1.0f + n + threadIdx.x * 1e-3f; }
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int n = 0; n < NACC; ++n) asm volatile("fma.rn.f32 %0, %1, %2, %0;" : "+f"(d[n]) : "f"(a[n]), "f"(h));
    }
    const long long t1 = clock64();
    float s = 0.f;
    for (int n = 0; n < NACC; ++n) s += d[n];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

int main() {
    float *out; long long *cyc;
    int nsm = 0;
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&out, nsm * 1024 * sizeof(float));
    cudaMalloc(&cyc, nsm * sizeof(long long));
    const int iters = 2000;
    for (int warps : {4, 8, 16}) {
        long long h[1];
        mma_kernel<8><<<nsm, warps * 32>>>(out, cyc, iters);
        cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
        double per = (double)h[0] / (iters * 8.0 * warps / 4.0);      // cycles per mma per SMSP
        printf("mma.sync m16n8k8 tf32: %2d warps/SM: %.2f cycles per mma per SMSP  -> %.0f MAC/clk/SM\n", warps, per, 4 * 1024.0 / per);
        ffma_kernel<8><<<nsm, warps * 32>>>(out, cyc, iters);
        cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
        per = (double)h[0] / (iters * 8.0 * warps / 4.0);
        printf("ffma                 : %2d warps/SM: %.2f cycles per ffma per SMSP  -> %.0f FMA/clk/SM\n", warps, per, 4 * 32.0 / per);
    }
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
