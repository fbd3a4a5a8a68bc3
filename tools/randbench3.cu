// Microbenchmark 3: does cudaLimitMaxL2FetchGranularity change the cost of touching 1 / 2 / 4 adjacent 32-B
// sectors of a random 128-B line with SEPARATE load instructions from one thread?
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
__device__ __forceinline__ void ld256(const void* p, uint32_t (&w)[8]) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8]; ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
}
__device__ __forceinline__ uint32_t mix(uint32_t h) { h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h; }
template <int NS>   // sectors of the line touched (1, 2, 4), separate instructions, issued back to back
__global__ void k(const uint4* __restrict__ tab, uint32_t line_mask, int iters, uint32_t* out) {
    uint32_t x = mix(blockIdx.x * blockDim.x + threadIdx.x + 11);
    uint32_t acc = 0;
    for (int i = 0; i < iters; ++i) {
        size_t line = x & line_mask;
        uint32_t w[NS][8];
#pragma unroll
        for (int s = 0; s < NS; ++s) ld256(tab + 8 * line + 2 * s, w[s]);
        uint32_t v = 0;
#pragma unroll
        for (int s = 0; s < NS; ++s) v ^= w[s][s];
        x = mix(x + v + i); acc += v;
    }
    if (acc == 0x12345678u) out[0] = acc;
}
template <int NS> void run(const uint4* tab, size_t bytes, uint32_t* out) {
    int iters = 64, blocks = [] { cudaDeviceProp p; cudaGetDeviceProperties(&p, 0); return p.multiProcessorCount; }() * 4, threads = 512;
    uint32_t mask = uint32_t(bytes / 128) - 1;
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k<NS><<<blocks, threads>>>(tab, mask, iters, out);
    cudaEventRecord(a); k<NS><<<blocks, threads>>>(tab, mask, iters, out); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    double lines = double(blocks) * threads * iters;
    printf("  %d sector(s) per random line, separate instr: %7.1f G lines/s  %.3f ms\n", NS, lines / ms / 1e6, ms);
}
int main() {
    size_t bytes = size_t(1) << 31;
    uint4* tab; cudaMalloc(&tab, bytes); cudaMemset(tab, 1, bytes);
    uint32_t* out; cudaMalloc(&out, 4);
    for (size_t g : {size_t(32), size_t(64), size_t(128)}) {
        cudaError_t e = cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, g);
        size_t got = 0; cudaDeviceGetLimit(&got, cudaLimitMaxL2FetchGranularity);
        printf("L2 fetch granularity requested %zu -> %zu (%s)\n", g, got, cudaGetErrorString(e));
        run<1>(tab, bytes, out); run<2>(tab, bytes, out); run<4>(tab, bytes, out);
    }
    return 0;
}
