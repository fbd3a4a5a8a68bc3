// Multi-GPU side of the path (SURVEY.md §8e, BASELINE.json C5): the subscription set is sharded by the hash of the
// topic root over the ranks (one process per GPU), a mixed PUBLISH batch is partitioned by the same hash ON THE
// DEVICE, every rank matches its share, and ONE all-gatherv makes every rank hold every topic's match list —
// the device-side analogue of results crossing nodes in rmqtt-cluster-raft/src/shared.rs:395-445.
//
// NCCL has no native all-gatherv: the collective is an ncclAllGather of the per-rank sizes (k topics, m ids)
// followed by ONE grouped launch of point-to-point transfers (every rank ncclSends its three arrays — topic index, spans,
// ids, straight out of the buffers the match kernels wrote — to every peer and ncclRecvs theirs into pre-sized contiguous
// arrays; over NVSwitch every pair has its own full-bandwidth path, so the pairs run at once instead of one broadcast
// root at a time); a small kernel re-bases the received spans.  libnccl is bound at run time (dlopen) so that the library loads, and everything single-GPU
// works, on hosts without NCCL; inside a torch process the already-loaded libnccl.so.2 is reused.
#pragma once
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <mutex>
#include <string>

#include "layout.h"

namespace gm {

struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int*) = nullptr;
    void* handle = nullptr;
    std::string error;

    static NcclApi& get() {
        static NcclApi api;
        static std::once_flag once;
        std::call_once(once, [] { api.load(); });
        return api;
    }
    bool ok() const { return handle != nullptr && error.empty(); }

  private:
    template <class F> void sym(F& f, const char* name) {
        f = reinterpret_cast<F>(dlsym(handle, name));
        if (!f && error.empty()) error = std::string("libnccl: missing symbol ") + name;
    }
    void load() {
        // a library with this SONAME that the process already holds (torch's bundled NCCL) wins
        for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
            handle = dlopen(name, RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
            if (!handle) handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (handle) break;
        }
        if (!handle) { error = std::string("libnccl.so.2 not found: ") + (dlerror() ? dlerror() : ""); return; }
        sym(GetUniqueId, "ncclGetUniqueId"); sym(CommInitRank, "ncclCommInitRank"); sym(CommDestroy, "ncclCommDestroy");
        sym(AllGather, "ncclAllGather"); sym(Broadcast, "ncclBroadcast"); sym(Send, "ncclSend"); sym(Recv, "ncclRecv"); sym(GroupStart, "ncclGroupStart"); sym(GroupEnd, "ncclGroupEnd");
        sym(GetErrorString, "ncclGetErrorString"); sym(GetVersion, "ncclGetVersion");
    }
};

// ------------------------------------------------------------------------------------------------
// Partition of a mixed batch: shard of every topic by its level-0 string — the SAME function the host uses to place
// filters (HostTrie::level0_hash -> shard_of_hash, gm_shard_of) — and compaction of this rank's topics into `sel`.
// Warp-aggregated append; the order inside `sel` is irrelevant (every row carries its global index).
// counts[r] receives the number of topics of shard r (load report); counts[nshards] = rows appended to sel.
constexpr u32 PART_SMEM_SHARDS = 1024;     // shard histograms up to this many shards are kept per CTA in shared memory
__global__ void __launch_bounds__(256)
k_partition(const u8* __restrict__ blob, u32 blob_bytes, const u32* __restrict__ offs, u32 n, u32 nshards, u32 rank, u32* __restrict__ sel,
            u32* __restrict__ shard_out, u32* __restrict__ counts) {
    __shared__ u32 s_hist[PART_SMEM_SHARDS];
    const bool smem_hist = nshards <= PART_SMEM_SHARDS;     // one global atomic per (CTA, shard) instead of one per topic
    if (smem_hist) { for (u32 i = threadIdx.x; i < nshards; i += blockDim.x) s_hist[i] = 0u; __syncthreads(); }
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    const u32 lane = threadIdx.x & 31;
    u32 shard = 0xFFFFFFFFu;
    if (t < n) {
        const u32 b = offs[t], e = min(offs[t + 1], blob_bytes);
        u32 h = FNV_INIT, l0 = 0;
        for (u32 i = b; i < e; ++i) {
            const u32 c = blob[i];
            if (c == '/') break;
            h = fnv_step(h, c);
            ++l0;
        }
        // a literal "+" / "#" root goes to shard 0 (any shard holds the replicated root wildcards; sharding.py partition_topics)
        const bool wild_root = l0 == 1 && (blob[b] == '+' || blob[b] == '#');
        shard = wild_root ? 0u : shard_of_hash(dict_hash_finish(h, l0), nshards);
        if (shard_out) shard_out[t] = shard;
        if (smem_hist) atomicAdd(s_hist + shard, 1u); else atomicAdd(counts + shard, 1u);
    }
    const bool mine = shard == rank;
    const u32 bal = __ballot_sync(0xFFFFFFFFu, mine);
    if (bal) {
        u32 base = 0;
        const int leader = __ffs(bal) - 1;
        if (static_cast<int>(lane) == leader) base = atomicAdd(counts + nshards, static_cast<u32>(__popc(bal)));
        base = __shfl_sync(0xFFFFFFFFu, base, leader);
        if (mine) sel[base + __popc(bal & ((1u << lane) - 1u))] = t;
    }
    if (smem_hist) {
        __syncthreads();
        for (u32 i = threadIdx.x; i < nshards; i += blockDim.x) { const u32 c = s_hist[i]; if (c) atomicAdd(counts + i, c); }
    }
}

// after the all-gatherv: spans of rank r's topics index rank r's id array; make them index the gathered array
__global__ void k_rebase_spans(uint2* __restrict__ spans, const unsigned long long* __restrict__ sizes /* [world][2] = (k, m) */, u32 world, u32 total_topics) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total_topics) return;
    unsigned long long ko = 0, mo = 0;
    for (u32 r = 0; r < world; ++r) {
        const unsigned long long k = sizes[2 * r], m = sizes[2 * r + 1];
        if (i < ko + k) break;
        ko += k; mo += m;
    }
    if (mo) { uint2 s = spans[i]; s.x += static_cast<u32>(mo); spans[i] = s; }
}

// PUSH form of the peer-memory gather: the match kernels published this rank's rows / ids into ITS OWN block; this kernel
// copies the slab to the same place in every peer's block with 16-byte loads and stores (NVLink writes in full 128-byte
// packets, every SM busy), still without a collective call or a host synchronisation.  The direct form (the publish
// phase storing every id into all blocks itself) stays selectable for comparison (debug knob gather_direct).
__global__ void __launch_bounds__(256)
k_gather_push(char* const* blocks /* [world] */, u32 rank, u32 world, size_t off_ids, size_t off_spans, size_t off_index,
              unsigned long long base_topics, unsigned long long base_ids, unsigned long long k, const unsigned long long* d_m) {
    const unsigned long long m = *d_m;
    const char* own = blocks[rank];
    // three byte ranges of the own block, each copied to every peer: ids, spans, index (starts are 16-byte aligned by layout)
    const size_t start[3] = {off_ids + base_ids * 4, off_spans + base_topics * 8, off_index + base_topics * 4};
    const size_t bytes[3] = {static_cast<size_t>(m) * 4, static_cast<size_t>(k) * 8, static_cast<size_t>(k) * 4};
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x, nth = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (int a = 0; a < 3; ++a) {
        const size_t lo = start[a] & ~size_t(15), hi = (start[a] + bytes[a] + 15) & ~size_t(15);      // whole 16-byte words (the slack belongs to this rank's slab)
        const size_t nvec = (hi - lo) / 16;
        const uint4* src = reinterpret_cast<const uint4*>(own + lo);
        for (size_t i = tid; i < nvec; i += nth) {
            const uint4 v = src[i];
            for (u32 w = 0; w < world; ++w) if (w != rank) reinterpret_cast<uint4*>(blocks[w] + lo)[i] = v;
        }
    }
}

#ifndef GM_CPU_EMU
__device__ __forceinline__ void st_release_sys(u32* p, u32 v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ u32 ld_acquire_sys(const u32* p) { u32 f; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(f) : "l"(p) : "memory"); return f; }
#else
inline void st_release_sys(u32* p, u32 v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
inline u32 ld_acquire_sys(const u32* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
#endif

// End of a fused-gather step: tell every rank how much this rank contributed and wait until every rank has said so —
// one warp, lane w talks to rank w.  The match kernels of this rank have completed (stream order), so its posted stores
// into the peers' buffers are performed before the release store of the flag; a rank that sees all flags of the epoch
// therefore sees all data.  A peer that never arrives (a failed rank) must not hang the GPU: the wait is bounded.
__global__ void k_gather_finish(unsigned long long* const* counts /* [world] peers' counts arrays [world][2] */, u32* const* flags /* [world] peers' flag arrays [world] */,
                                u32* my_flags, u32 rank, u32 world, unsigned long long k, const unsigned long long* d_m, u32 epoch, u32* err) {
    const u32 w = threadIdx.x;
    if (w >= world) return;
    counts[w][2 * rank] = k;
    counts[w][2 * rank + 1] = *d_m;
    __threadfence_system();
    st_release_sys(flags[w] + rank, epoch);
    const long long t0 = clock64();
    for (;;) {
        u32 f;
        f = ld_acquire_sys(my_flags + w);
        if (static_cast<int>(f - epoch) >= 0) break;
        if (clock64() - t0 > 6000000000ll) { atomicOr(err, 1u); break; }     // ~3 s at 2 GHz: give up, the host reports GM_ERR_COMM
        __nanosleep(200);
    }
}

// (k, m) of this rank into the send slot of the size exchange: m comes from the device cursor of the match
__global__ void k_comm_sizes(unsigned long long* out, unsigned long long k, const unsigned long long* d_m) {
    out[0] = k;
    out[1] = *d_m;
}

}  // namespace gm
