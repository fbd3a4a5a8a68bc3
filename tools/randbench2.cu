// Microbenchmark 2: random LINE fetches where G adjacent lanes of a warp load 32 B each from one aligned
// G*32-byte block with a single LDG.256 instruction (one L1 request, multi-sector mask).
// Question: is a random 64/128-byte block as cheap as a random 32-byte sector when requested at once?
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

__device__ __forceinline__ void ld256(const void* p, uint32_t (&w)[8]) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8]; ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
}
__device__ __forceinline__ uint32_t mix(uint32_t h) { h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h; }

template <int G>   // lanes per block: 1, 2, 4 (32, 64, 128 bytes)
__global__ void k(const uint4* __restrict__ tab, uint32_t nblocks_mask, int iters, uint32_t* out) {
    const uint32_t lane = threadIdx.x & 31, sub = lane % G, grp = (blockIdx.x * blockDim.x + threadIdx.x) / G;
    uint32_t x = mix(grp * 0x9E3779B1u + 7);
    uint32_t acc = 0;
    for (int i = 0; i < iters; ++i) {
        uint32_t w[8];
        size_t blk = x & nblocks_mask;                 // block index (G*32 bytes each)
        ld256(tab + 2 * (blk * G + sub), w);
        // next address must be identical for the G lanes of a group: take lane `sub==0`'s word
        uint32_t v = __shfl_sync(0xFFFFFFFFu, w[0], lane - sub);
        x = mix(x + v + i);
        acc += w[5];
    }
    if (acc == 0x12345678u) out[0] = acc;
}

template <int G>
void run(const uint4* tab, size_t bytes, uint32_t* out, const char* label) {
    int iters = 64, blocks = [] { cudaDeviceProp p; cudaGetDeviceProperties(&p, 0); return p.multiProcessorCount; }() * 4, threads = 512;
    uint32_t mask = uint32_t(bytes / (32 * G)) - 1;
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k<G><<<blocks, threads>>>(tab, mask, iters, out);
    cudaEventRecord(a);
    k<G><<<blocks, threads>>>(tab, mask, iters, out);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    double fetches = double(blocks) * threads / G * iters;
    printf("%-10s block=%3dB (1 instr, %d lanes): %7.1f G blocks/s  %7.1f GB/s  %.3f ms\n", label, 32 * G, G, fetches / ms / 1e6, fetches * 32 * G / ms / 1e6, ms);
}

int main() {
    for (int big = 0; big < 2; ++big) {
        size_t bytes = big ? (size_t(1) << 31) : (size_t(1) << 26);
        uint4* tab; cudaMalloc(&tab, bytes); cudaMemset(tab, 1, bytes);
        uint32_t* out; cudaMalloc(&out, 4);
        const char* label = big ? "DRAM 2GiB" : "L2 64MiB";
        run<1>(tab, bytes, out, label);
        run<2>(tab, bytes, out, label);
        run<4>(tab, bytes, out, label);
        cudaFree(tab); cudaFree(out);
    }
    return 0;
}
