// Microbenchmark 5: is the ~39 G/s ceiling on random 32-B fetches from a multi-GB table a DRAM limit or an
// address-translation (TLB) limit?  (a) uniform random over footprints 64 MiB .. 16 GiB; (b) the same number of
// cold DRAM fetches, but every CTA stays inside its own window of W bytes (few 2-MiB pages per SM, total
// footprint still >> L2).
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
__device__ __forceinline__ void ld256(const void* p, uint32_t (&w)[8]) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8]; ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
}
__device__ __forceinline__ uint32_t mix(uint32_t h) { h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h; }

// sectors: total 32-B sectors in the table (power of two); win_sectors: sectors per CTA window (power of two,
// == sectors for the uniform case).  The window base is a hash of (blockIdx, seed) aligned to the window size.
__global__ void k(const uint4* __restrict__ tab, uint64_t sectors, uint64_t win_sectors, int iters, uint32_t seed, uint32_t* out) {
    uint32_t x = mix((blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B1u + seed);
    const uint64_t nwin = sectors / win_sectors;
    const uint64_t base = (uint64_t(mix(blockIdx.x * 0x85EBCA77u + seed)) % nwin) * win_sectors;
    uint32_t acc = 0;
    for (int i = 0; i < iters; ++i) {
        uint64_t r = (uint64_t(x) << 20) ^ mix(x + 0x1234567u);
        uint64_t s = base + (r & (win_sectors - 1));
        uint32_t w[8];
        ld256(tab + 2 * s, w);
        x = mix(x + w[0] + i); acc += w[3];
    }
    if (acc == 0x12345678u) out[0] = acc;
}
static void run(const uint4* tab, size_t bytes, size_t win, uint32_t* out, const char* label) {
    int iters = 64, blocks = [] { cudaDeviceProp p; cudaGetDeviceProperties(&p, 0); return p.multiProcessorCount; }() * 4, threads = 512;
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k<<<blocks, threads>>>(tab, bytes / 32, win / 32, iters, 1u, out);
    cudaEventRecord(a); k<<<blocks, threads>>>(tab, bytes / 32, win / 32, iters, 2u, out); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    double n = double(blocks) * threads * iters;
    printf("  %-8s footprint %6zu MiB  window/CTA %6zu MiB: %6.1f G fetches/s  %.3f ms (%s)\n", label, bytes >> 20, win >> 20, n / ms / 1e6, ms,
           cudaGetErrorString(cudaGetLastError()));
}
int main() {
    size_t maxb = size_t(16) << 30;
    uint4* tab; if (cudaMalloc(&tab, maxb) != cudaSuccess) { printf("alloc failed\n"); return 1; }
    cudaMemset(tab, 1, maxb);
    uint32_t* out; cudaMalloc(&out, 4);
    for (size_t mb : {64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384}) run(tab, mb << 20, mb << 20, out, "uniform");
    for (size_t wmb : {2, 4, 8, 16, 32, 64, 128, 512}) run(tab, size_t(8) << 30, wmb << 20, out, "windowed");
    for (size_t wmb : {2, 8, 32, 128}) run(tab, size_t(16) << 30, wmb << 20, out, "windowed");
    return 0;
}
