// Microbenchmark 4: does the PTX prefetch-size hint (ld.global.L2::64B / L2::128B) turn the first miss on a random
// 128-B line into a whole-line fill, so that LATER loads of the neighbouring sectors (separate instructions,
// independent or data-dependent) become L2 hits instead of further miss requests?
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
template <int HINT> __device__ __forceinline__ void ld256(const void* p, uint32_t (&w)[8]) {
    if (HINT == 128)
        asm volatile("ld.global.nc.L2::128B.v4.u32 {%0,%1,%2,%3}, [%8]; ld.global.nc.L2::128B.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
    else if (HINT == 64)
        asm volatile("ld.global.nc.L2::64B.v4.u32 {%0,%1,%2,%3}, [%8]; ld.global.nc.L2::64B.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
    else
        asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8]; ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
}
__device__ __forceinline__ uint32_t mix(uint32_t h) { h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h; }

// NS sectors of one random line; sector 0 is loaded with the hint; DEP: each later sector's address depends on the
// data of the previous one (a pointer chase inside the line), else all NS loads are issued back to back.
template <int NS, int HINT, bool DEP>
__global__ void k(const uint4* __restrict__ tab, uint32_t line_mask, int iters, uint32_t* out) {
    uint32_t x = mix(blockIdx.x * blockDim.x + threadIdx.x + 11);
    uint32_t acc = 0;
    for (int i = 0; i < iters; ++i) {
        size_t line = x & line_mask;
        uint32_t v = 0;
        if (DEP) {
            uint32_t w[8];
            ld256<HINT>(tab + 8 * line, w);
            v = w[0];
#pragma unroll
            for (int s = 1; s < NS; ++s) {
                uint32_t sec = ((v >> 8) + s) & 3; if (sec == 0) sec = s;      // table is memset(1): sec == s, but unknown to the compiler
                ld256<0>(tab + 8 * line + 2 * sec, w);
                v ^= w[s];
            }
        } else {
            uint32_t w[NS][8];
            ld256<HINT>(tab + 8 * line, w[0]);
#pragma unroll
            for (int s = 1; s < NS; ++s) ld256<0>(tab + 8 * line + 2 * s, w[s]);
#pragma unroll
            for (int s = 0; s < NS; ++s) v ^= w[s][s];
        }
        x = mix(x + v + i); acc += v;
    }
    if (acc == 0x12345678u) out[0] = acc;
}
template <int NS, int HINT, bool DEP> void run(const uint4* tab, size_t bytes, uint32_t* out) {
    int iters = 64, blocks = [] { cudaDeviceProp p; cudaGetDeviceProperties(&p, 0); return p.multiProcessorCount; }() * 4, threads = 512;
    uint32_t mask = uint32_t(bytes / 128) - 1;
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k<NS, HINT, DEP><<<blocks, threads>>>(tab, mask, iters, out);
    cudaEventRecord(a); k<NS, HINT, DEP><<<blocks, threads>>>(tab, mask, iters, out); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    double lines = double(blocks) * threads * iters;
    printf("  %d sector(s)/line, hint %3d, %-11s: %6.1f G lines/s  %.3f ms  (%s)\n", NS, HINT, DEP ? "dependent" : "independent", lines / ms / 1e6, ms,
           cudaGetErrorString(cudaGetLastError()));
}
int main() {
    size_t bytes = size_t(1) << 31;
    uint4* tab; cudaMalloc(&tab, bytes); cudaMemset(tab, 1, bytes);
    uint32_t* out; cudaMalloc(&out, 4);
    run<1, 0, false>(tab, bytes, out); run<1, 64, false>(tab, bytes, out); run<1, 128, false>(tab, bytes, out);
    run<2, 0, false>(tab, bytes, out); run<2, 64, false>(tab, bytes, out); run<2, 128, false>(tab, bytes, out);
    run<4, 0, false>(tab, bytes, out); run<4, 128, false>(tab, bytes, out);
    run<2, 0, true>(tab, bytes, out);  run<2, 64, true>(tab, bytes, out);  run<2, 128, true>(tab, bytes, out);
    run<4, 0, true>(tab, bytes, out);  run<4, 128, true>(tab, bytes, out);
    return 0;
}
