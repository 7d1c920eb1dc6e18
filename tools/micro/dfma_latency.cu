// Microbenchmark: FP64 FMA issue cost per warp as a function of ILP (independent chains per thread)
// and warps per SM sub-partition.  Answers: what instruction latency must a 1-warp-per-scheduler
// kernel hide?   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dfma_latency dfma_latency.cu
#include <cstdio>
#include <cuda_runtime.h>
template <int ILP>
__global__ void chain(double* out, int iters, double a, double b) {
    double x[ILP];
#pragma unroll
    for (int k = 0; k < ILP; ++k) x[k] = threadIdx.x + k;
    long long t0 = clock64();
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < ILP; ++k) x[k] = fma(x[k], a, b);
    }
    long long t1 = clock64();
    double s = 0;
#pragma unroll
    for (int k = 0; k < ILP; ++k) s += x[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) reinterpret_cast<long long*>(out)[4096] = t1 - t0;
}
template <int ILP>
void run(int threads, double* d) {
    const int iters = 20000;
    chain<ILP><<<1, threads>>>(d, iters, 1.0000001, 1e-9);
    cudaDeviceSynchronize();
    long long cyc;
    cudaMemcpy(&cyc, reinterpret_cast<long long*>(d) + 4096, sizeof cyc, cudaMemcpyDeviceToHost);
    printf("warps/SM %2d  ILP %2d : %.2f cycles per DFMA per warp (%.2f cycles per loop iteration)\n", threads / 32, ILP,
           double(cyc) / (double(iters) * ILP), double(cyc) / iters);
}
int main() {
    double* d;
    cudaMalloc(&d, 1 << 20);
    for (int threads : {32, 128, 256, 512}) {
        run<1>(threads, d); run<2>(threads, d); run<4>(threads, d); run<8>(threads, d); run<16>(threads, d);
    }
    return 0;
}
