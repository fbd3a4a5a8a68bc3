// Microbenchmark for the "level-packed subtree + TMA bulk staging" layout the north-star text names (VERDICT r1 #4):
// how many RANDOM contiguous blocks per second can the GPU fetch from a multi-GB table when every block is requested by
// ONE cp.async.bulk (TMA engine -> shared memory), for block sizes 128 B .. 2 KB — against the same bytes fetched as
// per-lane 32-byte vector loads (what k_match_fast does today).  Answers: does fetching a packed ~0.3-1 KB subtree
// block with one bulk copy beat ~10 dependent 32-B probes?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o randbench6 randbench6.cu && ./randbench6
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <vector>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ uint32_t mix(uint32_t h) { h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h; }

// every WARP fetches `iters` random blocks of BLK bytes, DEPTH bulk copies in flight per warp (ring of mbarriers)
template <int BLK, int DEPTH>
__global__ void __launch_bounds__(256) k_bulk(const uint8_t* table, uint64_t nblocks, int iters, uint32_t* sink) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) unsigned long long bars[8 * DEPTH];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* stage = smem + static_cast<size_t>(warp) * DEPTH * BLK;
    unsigned long long* bar = bars + warp * DEPTH;
    if (lane == 0) for (int d = 0; d < DEPTH; ++d) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar + d)), "r"(1) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    uint32_t seed = mix((blockIdx.x * 8 + warp) * 0x9E3779B1u + 12345u), acc = 0;
    auto issue = [&](int d) {
        seed = mix(seed + 0x7F4A7C15u);
        const uint64_t b = (static_cast<uint64_t>(seed) * nblocks) >> 32;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar + d)), "r"(BLK) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(stage + d * BLK)), "l"(table + b * BLK), "r"(BLK), "r"(smem_u32(bar + d)) : "memory");
    };
    if (lane == 0) for (int d = 0; d < DEPTH; ++d) issue(d);
    for (int it = 0; it < iters; ++it) {
        const int d = it % DEPTH;
        const uint32_t parity = (it / DEPTH) & 1;
        uint32_t done = 0;
        while (!done) asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(done) : "r"(smem_u32(bar + d)), "r"(parity) : "memory");
        acc += reinterpret_cast<const uint32_t*>(stage + d * BLK)[lane % (BLK / 4)];      // consume
        __syncwarp();
        if (lane == 0 && it + DEPTH < iters) issue(d);
    }
    if (acc == 0xDEADBEEF) sink[0] = acc;
}

// baseline: every LANE fetches random 32-byte slots (two 128-bit loads each), `iters` per lane
__global__ void __launch_bounds__(256) k_lane32(const uint8_t* table, uint64_t nslots, int iters, uint32_t* sink) {
    uint32_t seed = mix((blockIdx.x * 256 + threadIdx.x) * 0x9E3779B1u + 999u), acc = 0;
    for (int it = 0; it < iters; ++it) {
        seed = mix(seed + 0x7F4A7C15u);
        const uint64_t s = (static_cast<uint64_t>(seed) * nslots) >> 32;
        uint32_t w[8];
        asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8]; ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(table + s * 32));
        acc += w[0] ^ w[7];
        seed ^= acc & 1;                      // dependent chain, like a trie walk
    }
    if (acc == 0xDEADBEEF) sink[0] = acc;
}

template <int BLK, int DEPTH>
void run_bulk(const uint8_t* table, uint64_t bytes, uint32_t* sink, int sms) {
    const int iters = 4096;
    const int grid = sms * 4;                 // 4 CTAs x 8 warps per SM
    const size_t smem = static_cast<size_t>(8) * DEPTH * BLK;
    cudaFuncSetAttribute(k_bulk<BLK, DEPTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k_bulk<BLK, DEPTH><<<grid, 256, smem>>>(table, bytes / BLK, 64, sink);
    cudaEventRecord(e0);
    k_bulk<BLK, DEPTH><<<grid, 256, smem>>>(table, bytes / BLK, iters, sink);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    const double blocks = double(grid) * 8 * iters;
    printf("{\"kind\": \"cp.async.bulk\", \"block_bytes\": %d, \"in_flight_per_warp\": %d, \"G_blocks_per_s\": %.2f, \"TB_per_s\": %.3f, \"err\": \"%s\"}\n", BLK, DEPTH,
           blocks / ms / 1e6, blocks * BLK / ms / 1e9, cudaGetErrorString(cudaGetLastError()));
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const uint64_t bytes = 8ull << 30;        // 8 GiB table >> L2
    uint8_t* table; uint32_t* sink;
    cudaMalloc(&table, bytes); cudaMalloc(&sink, 4);
    cudaMemset(table, 1, bytes);
    {
        const int iters = 512, grid = p.multiProcessorCount * 8;
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        k_lane32<<<grid, 256>>>(table, bytes / 32, 16, sink);
        cudaEventRecord(e0);
        k_lane32<<<grid, 256>>>(table, bytes / 32, iters, sink);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        const double n = double(grid) * 256 * iters;
        printf("{\"kind\": \"per-lane 2 x ld.global.v4 (32 B)\", \"block_bytes\": 32, \"G_blocks_per_s\": %.2f, \"TB_per_s\": %.3f}\n", n / ms / 1e6, n * 32 / ms / 1e9);
    }
    run_bulk<128, 8>(table, bytes, sink, p.multiProcessorCount);
    run_bulk<256, 8>(table, bytes, sink, p.multiProcessorCount);
    run_bulk<512, 8>(table, bytes, sink, p.multiProcessorCount);
    run_bulk<1024, 4>(table, bytes, sink, p.multiProcessorCount);
    run_bulk<2048, 2>(table, bytes, sink, p.multiProcessorCount);
    run_bulk<512, 2>(table, bytes, sink, p.multiProcessorCount);
    return 0;
}
