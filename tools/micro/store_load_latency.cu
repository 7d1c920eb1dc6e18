// Micro-benchmark behind the memory placement of the constraint solvers (DESIGN.md section 4): what does one thread
// of a lone warp pay to re-read a value it has just stored, in global / local / shared memory?
// Build + run: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/store_load_latency tools/micro/store_load_latency.cu && /tmp/store_load_latency
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ double ldg_(const double* p) { double v; asm volatile("ld.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void stg_(double* p, double v) { asm volatile("st.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
constexpr int N = 256;
__global__ void probe(double* buf, long long* out, double* sink) {
    extern __shared__ double sm[];
    if (threadIdx.x != 0) return;
    double acc = 1.0;
    long long t0, t1;
    const int stride = 32;   // doubles: one 256-byte step, a new line every access
    // 0. cold loads (HBM or L2, whatever the allocation left), dependent chain through the address
    t0 = clock64();
    for (int i = 0; i < N; ++i) { const int j = (static_cast<int>(acc) & 0) + i; acc += ldg_(buf + j * stride); }
    t1 = clock64(); out[0] = (t1 - t0) / N;
    // 1. same lines again: L1 hits if loads allocate
    t0 = clock64();
    for (int i = 0; i < N; ++i) { const int j = (static_cast<int>(acc) & 0) + i; acc += ldg_(buf + j * stride); }
    t1 = clock64(); out[1] = (t1 - t0) / N;
    // 2. store, then load the same address; the lines were loaded before (in L1 unless the store evicts them)
    t0 = clock64();
    for (int i = 0; i < N; ++i) { double* p = buf + i * stride; stg_(p, acc); acc = ldg_(p) + 1.0; }
    t1 = clock64(); out[2] = (t1 - t0) / N;
    // 3. store, then load the same address, on lines never touched by this SM
    double* fresh = buf + (1 << 20);
    t0 = clock64();
    for (int i = 0; i < N; ++i) { double* p = fresh + i * stride; stg_(p, acc); acc = ldg_(p) + 1.0; }
    t1 = clock64(); out[3] = (t1 - t0) / N;
    // 4. load the lines stored in 3. once more (did the store or the load after it allocate them?)
    t0 = clock64();
    for (int i = 0; i < N; ++i) { const int j = (static_cast<int>(acc) & 0) + i; acc += ldg_(fresh + j * stride); }
    t1 = clock64(); out[4] = (t1 - t0) / N;
    // 5. repeated store -> load on ONE address (the Gauss-Seidel pattern: the same few words updated over and over)
    t0 = clock64();
    for (int i = 0; i < N; ++i) { stg_(fresh, acc); acc = ldg_(fresh) + 1.0; }
    t1 = clock64(); out[5] = (t1 - t0) / N;
    // 6. local memory, dynamic index
    double loc[64];
    for (int i = 0; i < 64; ++i) loc[i] = acc + i;
    t0 = clock64();
    for (int i = 0; i < N; ++i) { const int j = (static_cast<int>(acc) & 63); int j2 = j; loc[j] = acc; asm volatile("" : "+r"(j2) :: "memory"); acc = loc[j2] + 1.0; }
    t1 = clock64(); out[6] = (t1 - t0) / N;
    // 7. shared memory
    t0 = clock64();
    for (int i = 0; i < N; ++i) { const int j = (static_cast<int>(acc) & 63); int j2 = j; sm[j] = acc; asm volatile("" : "+r"(j2) :: "memory"); acc = sm[j2] + 1.0; }
    t1 = clock64(); out[7] = (t1 - t0) / N;
    // 8. another thread of the same warp wrote it: covered by 2/3 (same L1)
    *sink = acc;
}
int main() {
    double* buf; long long* out; double* sink;
    cudaMalloc(&buf, (2 << 20) * sizeof(double)); cudaMemset(buf, 0, (2 << 20) * sizeof(double));
    cudaMallocManaged(&out, 16 * sizeof(long long)); cudaMalloc(&sink, 8);
    probe<<<1, 32, 64 * 8>>>(buf, out, sink);
    cudaDeviceSynchronize();
    const char* name[] = {"cold global load", "global load, second pass (L1 hit if loads allocate)", "store -> load, line already in L1",
                          "store -> load, line new to this SM", "reload of the lines of the previous test", "store -> load on one address, repeated",
                          "local memory store -> load (dynamic index)", "shared memory store -> load"};
    for (int i = 0; i < 8; ++i) printf("%-60s %6lld cycles\n", name[i], out[i]);
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
