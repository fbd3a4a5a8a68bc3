// Microbenchmark: how many random 32-byte sector loads per second does the GPU sustain?
// (the access pattern of the trie walk: one 32-byte load (two 128-bit halves) per visited node, dependent chains of length `chain`).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o randbench tools/randbench.cu
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

__device__ __forceinline__ void ld256(const void* p, uint32_t (&w)[8]) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8]; ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
}
__device__ __forceinline__ uint32_t mix(uint32_t h) { h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h; }

// each thread: `iters` dependent steps, each step issues MLP independent random loads whose results feed the next addresses
template <int MLP, int GRAN>   // GRAN = 1: one 32-B sector, 2: both sectors of a 64-B pair
__global__ void k(const uint4* __restrict__ tab, uint32_t mask, int iters, uint32_t* out) {
    uint32_t x[MLP];
    for (int j = 0; j < MLP; ++j) x[j] = mix(blockIdx.x * blockDim.x + threadIdx.x + j * 0x9E3779B1u);
    uint32_t acc = 0;
    for (int i = 0; i < iters; ++i) {
        uint32_t w[MLP][8];
#pragma unroll
        for (int j = 0; j < MLP; ++j) {
            size_t slot = (x[j] & mask);
            if (GRAN == 2) slot &= ~size_t(1);
            ld256(tab + 2 * slot, w[j]);
            if (GRAN == 2) { uint32_t w2[8]; ld256(tab + 2 * slot + 2, w2); w[j][0] ^= w2[3]; }
        }
#pragma unroll
        for (int j = 0; j < MLP; ++j) { x[j] = mix(x[j] + w[j][0] + i); acc += w[j][5]; }
    }
    if (acc == 0x12345678u) out[0] = acc;
}

template <int MLP, int GRAN>
void run(const uint4* tab, uint32_t mask, uint32_t* out, int blocks, int threads, const char* label) {
    int iters = 64;
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k<MLP, GRAN><<<blocks, threads>>>(tab, mask, iters, out);
    cudaEventRecord(a);
    k<MLP, GRAN><<<blocks, threads>>>(tab, mask, iters, out);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    double loads = double(blocks) * threads * iters * MLP;
    printf("%-10s MLP=%d gran=%dB threads/SM=%4d : %7.1f G loads/s  %7.1f GB/s (requested)  %.3f ms\n", label, MLP, 32 * GRAN, blocks / [] { cudaDeviceProp p; cudaGetDeviceProperties(&p, 0); return p.multiProcessorCount; }() * threads, loads / ms / 1e6, loads * 32 * GRAN / ms / 1e6, ms);
}

int main() {
    const int sms = [] { cudaDeviceProp p; cudaGetDeviceProperties(&p, 0); return p.multiProcessorCount; }();
    for (int big = 0; big < 2; ++big) {
        size_t slots = big ? (size_t(1) << 26) : (size_t(1) << 20);     // 2 GiB (DRAM) / 32 MiB (L2-resident on a 50 MB L2)
        uint4* tab; cudaMalloc(&tab, slots * 32); cudaMemset(tab, 1, slots * 32);
        uint32_t* out; cudaMalloc(&out, 4);
        const char* label = big ? "DRAM 2GiB" : "L2 32MiB";
        run<1, 1>(tab, slots - 1, out, sms * 4, 512, label);
        run<1, 1>(tab, slots - 1, out, sms * 2, 512, label);
        run<2, 1>(tab, slots - 1, out, sms * 4, 512, label);
        run<4, 1>(tab, slots - 1, out, sms * 4, 512, label);
        run<8, 1>(tab, slots - 1, out, sms * 2, 512, label);
        run<1, 2>(tab, slots - 1, out, sms * 4, 512, label);
        run<4, 2>(tab, slots - 1, out, sms * 4, 512, label);
        cudaFree(tab); cudaFree(out);
    }
    return 0;
}
