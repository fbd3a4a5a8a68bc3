// sm_90a kernels of the PUBLISH -> matching-subscribers hot path.
//
//   k_tokenize     Topic::from_str (rmqtt/src/topic.rs:326-363) for a batch: split on '/', classify,
//                  validate, and intern every level through the device dictionary -> u32 tokens.
//   k_match_fast   TopicTree::matches (rmqtt/src/trie.rs:299-347, MatchedIter::prepare): one topic per
//                  thread walks the trie depth-first (one 32-byte load per visited node), then the warp
//                  reserves its 32 match lists (per-topic contiguous output) and records their value sets.
//   k_match_expand writes the ids of those value sets with a load-balanced (scan / shuffle search) copy.
//   k_match_slow   the same walk for the topics the fast path defers (more levels than the fast
//                  path stages in shared memory, or more matches than its staging pool): one warp per
//                  topic, count pass + write pass, warp-cooperative value-range copies.
//   k_apply_patches  flush of 32-byte slot patches into the device tables (Router::add/remove).
//
// All arithmetic is u32 integer / pointer chasing: HBM- and L2-latency bound; no tensor cores.
#pragma once
#include <cuda_runtime.h>

#include "layout.h"

// a kernel launch; the CPU emulation (tests/native/emu, -DGM_CPU_EMU) runs the same kernel over host memory
#ifdef GM_CPU_EMU
#define GM_LAUNCH(k, grid, block, smem, s, ...) emu::launch(dim3(grid), dim3(block), [&] { k(__VA_ARGS__); })
#else
#define GM_LAUNCH(k, grid, block, smem, s, ...) k<<<grid, block, smem, s>>>(__VA_ARGS__)
#endif

namespace gm {

struct MatchParams {
    TrieView tv;
    const u32* tok8;     // [n][8]  tokens of levels 0..7, one 32-byte row per topic (one 32-byte load)
    const u32* tok;      // [tok_levels][n]  levels >= 8 only (level-major; deferred kernel)
    const u32* meta;     // [n]
    u32 n;
    u32 tok_levels;
    uint2* spans;        // [n] (offset, count) into out_ids
    u32* out_ids;
    unsigned long long cap_ids;
    unsigned long long* cursor;   // bump allocator over out_ids (final value = ids needed)
    u32* slow_list;      // [n]
    u32* slow_count;
    u32* tile_counter;
    unsigned long long* stats;    // [4] V,E,F,M + [4..] probe diagnostics (only written by STATS instantiations)
    u32 flags;                    // MP_* tuning switches
    const u32* perm;     // [n] locality order (k_bucket_*): position -> topic index
    const u32* tok8_sorted;   // [n][8] token rows copied into locality order (MP_SORTED_ROWS)
    const u32* meta_sorted;   // [n]
    u32 tile_chunk;           // tiles a CTA takes from the global counter at once (<= 1: one tile per warp per grab)
    // FUSED GATHER (peer memory): the match writes every result DIRECTLY into the gathered buffers of all ranks (own
    // included) over NVLink — no separate collective; spans and indices as the walk goes, ids from k_match_expand.  Rank r's rows
    // occupy the fixed slab [r * slab_topics, ...) / ids [r * slab_ids, ...) of every rank's buffers.
    u32* g_ids[8];            // gathered id arrays of ranks 0..g_world-1 (peer pointers, CUDA IPC)
    uint2* g_spans[8];
    u32* g_index[8];
    u32 g_world;              // 0 = off
    u32 g_base_topics;        // this rank's slab start, in rows
    unsigned long long g_base_ids;   // ... and in ids
    const u32* g_sel;         // row -> global topic index (the selection of gm_partition_batch_device), null: identity
    const u32* trees;         // [n] optional: the tree every row is matched against (0 = the subscription trie)
    const u32* n_ptr;         // small-batch graphs: the real batch size lives in device memory (n is then the capacity = row stride of `tok`)
    uint2* out_desc;          // DESCRIPTOR mode: matched value sets (ref, cnt16) per topic instead of expanded ids; spans index this array
    int* status;              // [n] per-topic status (k_tokenize wrote it); the deferred kernel reports GM_ERR_INTERNAL here
    // ids mode: k_match_fast stores the matched value sets (ref, cnt) of every tile whose ids fit into `items`, in the order of
    // their ids, and one record per tile; k_match_expand turns them into ids
    uint2* items;
    struct TileRec* tiles;    // [ceil(n / 32)], indexed by tile
    unsigned long long* item_cursor;   // bump allocator over `items`
};
// where k_match_expand finds a tile's value sets and writes its ids (n_items = 0: nothing to write)
struct TileRec { u32 item_base, n_items; unsigned long long id_base; };
static_assert(sizeof(TileRec) == 16, "one 16-byte record per tile");
constexpr u32 MP_DIAG_NO_PUBLISH = 2u;   // diagnostics only: the fast path writes no ids (k_match_fast records no value sets for k_match_expand; k_match_slow still writes the deferred topics' ids)
constexpr u32 MP_SORTED_ROWS = 1u;   // k_bucket_scatter also copies token rows + meta into sorted order (coalesced reads in k_match_fast)
constexpr u32 MAX_BUCKET_BITS = 18;   // locality buckets: 2^bits, bits = site_bits + sub_bits (engine.cu)
constexpr u32 TOK8 = 8;              // levels kept in the per-topic 32-byte token row
constexpr u32 K2_SMEM_DESCS = 8;     // value-set descriptors per topic held in shared memory by k_match_fast
template <int FAST_L, int THREADS> constexpr size_t k2_smem_bytes() { return (2 * sizeof(u32) * FAST_L + sizeof(uint2) * K2_SMEM_DESCS) * THREADS; }

// ------------------------------------------------------------------------------------------------
// (GM_CPU_EMU: tests/native/emu runs these kernels on the CPU under the sanitizers — the few PTX helpers have plain C++ twins)
#ifndef GM_CPU_EMU
// One 32-byte slot (32-byte aligned).  sm_90 has no 256-bit access: two 128-bit halves, issued back to back, which
// fall into the same 32-byte L2 sector, so a slot still costs one sector of DRAM traffic.
__device__ __forceinline__ void ld256(const void* p, u32 (&w)[8]) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
                 : "l"(p));
}
__device__ __forceinline__ void st256(void* p, const u32 (&w)[8]) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};\n\t"
                 "st.global.v4.u32 [%0+16], {%5,%6,%7,%8};" ::"l"(p), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]), "r"(w[4]), "r"(w[5]), "r"(w[6]), "r"(w[7]) : "memory");
}
__device__ __forceinline__ u32 lanemask_lt() {
    u32 m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}
#else
inline void ld256(const void* p, u32 (&w)[8]) { __builtin_memcpy(w, p, 32); }
inline void st256(void* p, const u32 (&w)[8]) { __builtin_memcpy(p, w, 32); }
inline u32 lanemask_lt() { return (1u << (threadIdx.x & 31u)) - 1u; }
#endif

// ------------------------------------------------------------------------------------------------
// K1: tokeniser.  One thread per topic, FOUR text bytes per step: the level text is read with aligned
// 32-bit loads re-aligned by a funnel shift, '/' and the wildcard characters are found with SWAR zero-byte
// tests, and the packed key words of the level stay in registers (static indexing) where they are compared
// directly with the 32-byte dictionary slot.  (A byte-at-a-time loop packing through shared memory spends many
// instructions per text byte and is issue bound.)
constexpr int TOK_THREADS = 256;

__device__ __forceinline__ u32 swar_zero_bytes(u32 v) { return (v - 0x01010101u) & ~v & 0x80808080u; }   // bit 7 of every zero byte (lowest hit exact)

// four text bytes starting at byte address `a` (little endian); never dereferences at or beyond `limit`
__device__ __forceinline__ u32 text4(const u8* a, const u8* limit) {
    const uintptr_t ai = reinterpret_cast<uintptr_t>(a);
    const u32* w = reinterpret_cast<const u32*>(ai & ~uintptr_t(3));
    const u32 lo = reinterpret_cast<const u8*>(w) < limit ? __ldg(w) : 0u;
    const u32 hi = reinterpret_cast<const u8*>(w + 1) < limit ? __ldg(w + 1) : 0u;
    return __funnelshift_r(lo, hi, 8u * static_cast<u32>(ai & 3));
}

// the same out of the CTA's shared-memory stage of the text slice (`sbase` = blob offset of stage byte 0, 16-byte aligned;
// the stage is zero-padded past the copied bytes up to its capacity, so whole-word reads are always defined)
__device__ __forceinline__ u32 text4_s(const u32* stage, u32 off) {
    const u32 lo = stage[off >> 2], hi = stage[(off >> 2) + 1];
    return __funnelshift_r(lo, hi, 8u * (off & 3u));
}

// ---- 1-D bulk asynchronous copy global -> shared (TMA engine, cp.async.bulk), completion on an mbarrier ----------------
#ifndef GM_CPU_EMU
__device__ __forceinline__ u32 smem_u32(const void* p) { return static_cast<u32>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, u32 bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, u32 parity) {
    u32 done = 0;
    while (!done) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    }
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
#else      // the bulk copy completes at once; the barrier has nothing to wait for
inline void mbar_init(unsigned long long*, u32) {}
inline void mbar_expect_tx(unsigned long long*, u32) {}
inline void bulk_g2s(void* dst_smem, const void* src_gmem, u32 bytes, unsigned long long*) { __builtin_memcpy(dst_smem, src_gmem, bytes); }
inline void mbar_wait(unsigned long long*, u32) {}
inline void mbar_fence_init() {}
#endif

__device__ __forceinline__ u32 dict_lookup_inline(const TrieView& tv, const u32 (&w)[7]) {
    u32 idx = dict_hash_words(w) & tv.dict_mask;
    for (;;) {
        u32 s[8];
        ld256(tv.dict + idx, s);
        if (s[0] == 0) return TOK_UNKNOWN;
        bool eq = true;
#pragma unroll
        for (int k = 0; k < 7; ++k) eq &= (s[k + 1] == w[k]);
        if (eq) return s[0];
        idx = (idx + 1) & tv.dict_mask;
    }
}

// (a template only so that every kernel instantiation owns its private out-of-line copy: two kernels sharing one
//  noinline function made ptxas 12.9 crash once one of them used the bulk-copy / mbarrier instructions)
template <int OWNER>
__device__ __noinline__ u32 dict_lookup_long(const TrieView& tv, const u8* text, u32 len) {
    u32 h = FNV_INIT;
    for (u32 i = 0; i < len; ++i) h = fnv_step(h, text[i]);
    u32 idx = dict_hash_finish(h, len) & tv.dict_mask;
    for (;;) {
        u32 s[8];
        ld256(tv.dict + idx, s);
        if (s[0] == 0) return TOK_UNKNOWN;
        if ((s[7] >> 24) == 0xFFu && s[1] == len && s[3] == h) {
            const u8* q = tv.pool + s[2];
            bool eq = true;
            for (u32 i = 0; i < len && eq; ++i) eq = (q[i] == text[i]);
            if (eq) return s[0];
        }
        idx = (idx + 1) & tv.dict_mask;
    }
}

// `sel` (optional): row t tokenises entry sel[t] of the packed batch (this rank's topics of a mixed batch, gm_partition_batch_device).
// `blob_bytes` bounds every text read: words that start at or beyond blob + blob_bytes are never dereferenced.
// BULK: the CTA's 256 topics are one contiguous slice of the blob (~12 KB on C3).  One elected thread asks the TMA engine
// for the whole slice with ONE cp.async.bulk into shared memory (16-byte aligned superset of the slice, completion
// counted in bytes on an mbarrier) and every thread then reads its topic's text from shared memory, instead of every
// thread pulling its own unaligned 32-bit words through L1.  `readable_bytes` (>= blob_bytes) says how far the
// allocation may be read; a CTA whose aligned slice does not fit the stage or the readable range, a blob pointer that is
// not 16-byte aligned, or a selection (`sel`: rows are not contiguous) takes the plain global-load path.
constexpr u32 TOK_STAGE_BYTES = 24 * 1024;    // 96 B per topic on average before a CTA falls back
template <bool BULK>
__global__ void __launch_bounds__(TOK_THREADS)
k_tokenize(const u8* __restrict__ blob, u32 blob_bytes, u32 readable_bytes, const u32* __restrict__ offs, const u32* __restrict__ sel, u32 n, const u32* __restrict__ hdr, TrieView tv, u32 tok_levels,
           u32* __restrict__ tok8, u32* __restrict__ tok, u32* __restrict__ meta, int* __restrict__ status, u32* __restrict__ bkey,
           u32* __restrict__ hist, u32 site_bits, u32 sub_bits) {
    __shared__ __align__(128) u32 s_stage[BULK ? TOK_STAGE_BYTES / 4 + 2 : 1];
    __shared__ __align__(8) unsigned long long s_bar;
    // small-batch graphs: the launch is sized for a CAPACITY `n`; the real batch size and text length sit in device memory
    const u32 stride = n;                        // row stride of the level-major `tok` array
    if (hdr) { n = min(n, hdr[0]); blob_bytes = readable_bytes = hdr[1]; }
    bool staged = false;
    u32 sbase = 0;
    if (BULK) {
        const u32 t0 = blockIdx.x * TOK_THREADS, t1 = min(n, t0 + TOK_THREADS);
        const bool any = t0 < n;                 // (a capacity-sized launch has CTAs beyond the real batch)
        const u32 b0 = any ? offs[t0] & ~15u : 0u;
        const u32 e0 = any ? (min(offs[t1], blob_bytes) + 15u) & ~15u : 0u;
        staged = any && sel == nullptr && (reinterpret_cast<uintptr_t>(blob) & 15u) == 0 && e0 > b0 && e0 - b0 <= TOK_STAGE_BYTES && e0 <= readable_bytes;
        if (staged) {           // uniform over the CTA
            sbase = b0;
            if (threadIdx.x == 0) {
                mbar_init(&s_bar, 1);
                mbar_fence_init();
                mbar_expect_tx(&s_bar, e0 - b0);
                bulk_g2s(s_stage, blob + b0, e0 - b0, &s_bar);
            }
            // the two words behind the copied bytes are read by text4_s of the last topic: define them
            if (threadIdx.x == 1) { s_stage[(e0 - b0) >> 2] = 0u; s_stage[((e0 - b0) >> 2) + 1] = 0u; }
            __syncthreads();    // barrier initialised before anyone polls it
            mbar_wait(&s_bar, 0);
        }
    }
    const u32 t = blockIdx.x * TOK_THREADS + threadIdx.x;
    if (t >= n) return;
    const u32 src = sel ? sel[t] : t;
    u32 pos = offs[src];
    const u32 end = min(offs[src + 1], blob_bytes);
    const u8* limit = blob + blob_bytes;
    u32 lev = 0;
    u32 tw[TOK8] = {0, 0, 0, 0, 0, 0, 0, 0};   // tokens of levels 0..7 (static indexing only: stays in registers)
    bool invalid = false, dollar = false;
    for (;;) {
        const u32 start = pos;
        u32 w[7] = {0, 0, 0, 0, 0, 0, 0};
        u32 len = 0;
        bool ended = false, wild = false;
#pragma unroll
        for (int k = 0; k < 7; ++k) {
            if (!ended) {
                u32 x = (BULK && staged) ? text4_s(s_stage, pos - sbase) : text4(blob + pos, limit);
                const u32 z = swar_zero_bytes(x ^ 0x2F2F2F2Fu);                       // '/' bytes
                u32 nb = z ? static_cast<u32>((__ffs(z) - 1) >> 3) : 4u;             // bytes before the first '/'
                nb = min(nb, end - pos);                                             // ... and before the end of the topic
                ended = nb < 4;
                x &= nb == 4 ? 0xFFFFFFFFu : ((1u << (8 * nb)) - 1u);
                wild |= (swar_zero_bytes(x ^ 0x2B2B2B2Bu) | swar_zero_bytes(x ^ 0x23232323u)) != 0;   // '+' / '#'
                w[k] = x;
                len += nb; pos += nb;
            }
        }
        if (!ended) {   // 28 bytes and still inside the level: long level (rare) — finish byte-wise
            while (pos < end && blob[pos] != '/') { const u32 c = blob[pos]; wild |= (c == '+') | (c == '#'); ++pos; ++len; }
        }
        const u32 c0 = w[0] & 0xFFu;
        const bool last = pos >= end;
        u32 tk = TOK_UNKNOWN;
        if (len == 0) tk = TOK_BLANK;
        else if (len == 1 && c0 == '+') tk = TOK_PLUS;
        else if (len == 1 && c0 == '#') { tk = TOK_HASH; if (!last) invalid = true; }   // topic.rs:209
        else if (wild) invalid = true;                                                   // topic.rs:333-334
        else {
            if (c0 == '$') { if (lev > 0) invalid = true; else dollar = true; }           // topic.rs:210
            if (!invalid && lev < tok_levels) {
                if (len <= DICT_INLINE_MAX) { w[6] |= len << 24; tk = dict_lookup_inline(tv, w); }
                else tk = dict_lookup_long<BULK ? 1 : 0>(tv, blob + start, len);
            }
        }
        if (invalid) break;
#pragma unroll
        for (u32 k = 0; k < TOK8; ++k) if (lev == k) tw[k] = tk;
        if (lev >= TOK8 && lev < tok_levels) tok[static_cast<size_t>(lev) * stride + t] = tk;
        ++lev;
        if (last) break;
        ++pos;   // skip '/'
    }
    meta[t] = invalid ? META_INVALID : (lev | (dollar ? META_DOLLAR : 0u));
    status[t] = invalid ? -2 : 0;   // GM_ERR_INVALID_TOPIC: Topic::from_str would return Err
    st256(tok8 + static_cast<size_t>(t) * TOK8, tw);
    if (bkey) {   // locality bucket: topics that share their first two levels share the upper subtrees of the trie
        // major key: the first two levels (shared upper subtrees); minor key: a few bits of the third (neighbouring
        // tiles then also share the cold per-device chains when a device shows up more than once in the batch)
        const u32 b = invalid ? 0u : (((fmix32(tw[0] * 0x9E3779B1u + tw[1]) & ((1u << site_bits) - 1u)) << sub_bits) | (fmix32(tw[2]) & ((1u << sub_bits) - 1u)));
        bkey[t] = b;
        atomicAdd(hist + b, 1u);
    }
}

// ------------------------------------------------------------------------------------------------
// Locality pass.  A uniformly random batch revisits a shared subtree (say the filters below `reg/site/+`)
// once every few thousand topics — long enough for the cold random stream to evict it from L2 in between.
// Regrouping the batch by hash(level 0, level 1) makes the topics that
// share those subtrees run in the same tiles: the second and later visits hit L1/L2.  Counting sort:
// histogram (in k_tokenize) -> k_bucket_scan -> k_bucket_scatter; order inside a bucket is irrelevant.
__global__ void __launch_bounds__(1024)
k_bucket_scan(const u32* __restrict__ hist, u32* __restrict__ cursor, u32 nbuckets) {
    __shared__ u32 s_warp[32];
    // thread t owns the 128-bit words [t*per4, (t+1)*per4) of the histogram; nbuckets is a power of two >= 1024
    const u32 per4 = max(nbuckets / 4096u, 1u);
    const u32 tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const bool mine = static_cast<size_t>(tid) * per4 * 4 < nbuckets;
    const uint4* __restrict__ h4 = reinterpret_cast<const uint4*>(hist) + static_cast<size_t>(tid) * per4;
    u32 sum = 0;
    if (mine)
        for (u32 k = 0; k < per4; ++k) { const uint4 v = h4[k]; sum += v.x + v.y + v.z + v.w; }
    u32 inc = sum;                                   // warp-level inclusive scan by shuffle
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { u32 x = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= o) inc += x; }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        u32 w = s_warp[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { u32 x = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= o) wi += x; }
        s_warp[lane] = wi - w;                        // exclusive offset of each warp
    }
    __syncthreads();
    if (!mine) return;
    u32 run = s_warp[wid] + inc - sum;
    uint4* __restrict__ c4 = reinterpret_cast<uint4*>(cursor) + static_cast<size_t>(tid) * per4;
    for (u32 k = 0; k < per4; ++k) {
        const uint4 v = h4[k];
        uint4 o;
        o.x = run; run += v.x; o.y = run; run += v.y; o.z = run; run += v.z; o.w = run; run += v.w;
        c4[k] = o;
    }
}

__global__ void __launch_bounds__(256)
k_bucket_scatter(const u32* __restrict__ bkey, u32* __restrict__ cursor, u32 n, const u32* __restrict__ hdr, u32* __restrict__ perm,
                 const u32* __restrict__ tok8, const u32* __restrict__ meta, u32* __restrict__ tok8_sorted, u32* __restrict__ meta_sorted) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (hdr) n = min(n, hdr[0]);
    if (t >= n) return;
    const u32 pos = atomicAdd(cursor + bkey[t], 1u);
    perm[pos] = t;
    if (tok8_sorted) {
        u32 w[8];
        ld256(tok8 + static_cast<size_t>(t) * TOK8, w);
        st256(tok8_sorted + static_cast<size_t>(pos) * TOK8, w);
        meta_sorted[pos] = meta[t];
    }
}

// ------------------------------------------------------------------------------------------------
// Work items.  lo = argument (parent node id for a literal probe, 1 + edge slot of the '+' child for a '+' hop),
// hi = topic slot (5 bits) | depth of the node being loaded << 5 | kind << 21 | window tag of the parent << 22.
constexpr u32 KIND_PROBE = 0, KIND_PLUS = 1;
__device__ __forceinline__ u64 make_item(u32 topic, u32 depth, u32 kind, u32 arg, u32 wtag = 0u) {
    return (static_cast<u64>(topic | (depth << 5) | (kind << 21) | (wtag << 22)) << 32) | arg;
}

struct NodeRec { u32 node, plus, hash_ref, own_ref, mask, cnts; };

// Loads the record an item points at.  Returns false when the literal child does not exist.
// `pmask_tag`: the mask word of the PARENT's record — its top byte names the window holding the parent's child edges.
__device__ __forceinline__ bool load_record(const TrieView& tv, u32 kind, u32 arg, u32 token, u32 pmask_tag, NodeRec& r) {
    u32 s[8];
    if (kind == KIND_PLUS) {                               // arg = 1 + slot of the '+' child: no hashing, no key compare
        ld256(tv.edges + (arg - 1u), s);
        r.node = s[2]; r.plus = s[3]; r.hash_ref = s[4]; r.own_ref = s[5]; r.mask = s[6]; r.cnts = s[7];
        return true;
    }
    u32 idx = edge_slot0(arg, token, pmask_tag >> WTAG_SHIFT, tv.win_mask, tv.win_shift, tv.nwin_mask);
    for (;;) {
        ld256(tv.edges + idx, s);
        if (s[2] == 0) return false;                       // empty slot: no such child
        if (s[0] == arg && s[1] == token) break;
        idx = edge_next(idx, tv.win_mask);
    }
    r.node = s[2]; r.plus = s[3]; r.hash_ref = s[4]; r.own_ref = s[5]; r.mask = s[6]; r.cnts = s[7];
    return true;
}

// child filter of wide nodes (layout.h): false = the child certainly does not exist
__device__ __forceinline__ bool cfilter_maybe(const TrieView& tv, u32 parent, u32 token) {
    u32 w, bits;
    cfilter_pos(parent, token, tv.cfilter_mask, w, bits);
    return (__ldg(tv.cfilter + w) & bits) == bits;
}

// Tile scheduling.  Tiles are in locality order; handing them out one by one from a global counter scatters
// neighbouring tiles over all SMs.  Instead a CTA reserves `chunk` consecutive tiles at a time and its warps take
// them from shared memory, so the warps of one SM work on neighbouring (level0, level1) subtrees at the same time:
// shared upper-level slots hit L1/L2 and the cold probes of the SM stay inside few windows of the edge table.
// s_chunk = next tile (low word) | end of the reserved run (high word); s_lock serialises refills.  No barrier:
// a warp that finds the run exhausted either refills it (lock holder) or spins for the few hundred ns that takes.
__device__ __forceinline__ u32 next_tile_chunked(unsigned long long* s_chunk, u32* s_lock, u32* gcounter, u32 chunk) {
    for (;;) {
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(s_chunk);
        if (static_cast<u32>(cur) < static_cast<u32>(cur >> 32)) {
            if (atomicCAS(s_chunk, cur, cur + 1ull) == cur) return static_cast<u32>(cur);
            continue;
        }
        if (atomicCAS(s_lock, 0u, 1u) == 0u) {
            cur = *reinterpret_cast<volatile unsigned long long*>(s_chunk);
            if (static_cast<u32>(cur) < static_cast<u32>(cur >> 32)) { atomicExch(s_lock, 0u); continue; }   // refilled in between
            const u32 base = atomicAdd(gcounter, chunk);
            atomicExch(s_chunk, (static_cast<unsigned long long>(base + chunk) << 32) | (base + 1u));
            __threadfence_block();
            atomicExch(s_lock, 0u);
            return base;
        }
    }
}

// A matched value set waiting to be expanded into the output: values[ref .. ref+cnt) (or ref itself).
struct Desc { u32 ref, cnt; };

// Load-balanced expansion of a warp's 32 runs laid end to end (run lengths scanned into `exc`, the exclusive prefix): the
// lane whose run holds flat index e, by binary search over `exc` — the last lane whose run starts at or before e (an
// empty run starts where the next one does, so it never owns an index below the total).
__device__ __forceinline__ u32 warp_run_owner(u32 exc, u32 e) {
    u32 lo = 0;
#pragma unroll
    for (int step = 16; step; step >>= 1) {
        const u32 v = __shfl_sync(0xFFFFFFFFu, exc, lo + step);
        if (v <= e) lo += step;
    }
    return lo;
}

// K2: TopicTree::matches, one topic per thread (depth-first), one tile of 32 topics per warp.
//
//   walk     every thread follows its own topic down the trie: at a node it records the matched value
//            sets ('#' child always, own values on path exhaustion) as 8-byte descriptors, parks the
//            '+' child of this depth in its shared-memory column, and descends through the literal
//            child with ONE 32-byte load; when the literal path ends it resumes the deepest parked
//            '+' child.  The dependent chain of a thread is one load long per visited node; latency is
//            hidden by the other ~1.5 K resident threads of the SM.
//   publish  warp-cooperative: per-lane totals -> warp scan -> one atomic reservation of the tile's ids ->
//            the tile's descriptors, lane-major, into the item array and one TileRec per tile.  The ids
//            themselves are written by k_match_expand: expanding them here kept each warp away from the
//            walk for a long serial chain of shuffles and scattered stores, and the walk is latency bound.
//
// (A warp-shared ballot-compacted frontier queue instead is bound by its collective overhead, not by memory.)
// DESC = descriptor mode: the publish phase writes each topic's matched value-set references (ref, cnt16) — 8 bytes per
// matched FILTER instead of 4 bytes per matched id — and spans / cursor / cap count descriptors.  The host resolves
// them against its mirror of `values` (gm_desc_resolve): this is what DefaultRouter::_matches consumes anyway, one
// relations entry per matched filter (rmqtt/src/router.rs:166-182), and it cuts the D2H volume ~4x.
template <int FAST_L, int THREADS, int CTAS_PER_SM, bool STATS, bool DESC, bool GATHER = false>
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM)
k_match_fast(MatchParams p, Desc* __restrict__ dpool, u32 pool_rows) {
    static_assert(!(GATHER && DESC), "the fused gather publishes ids");
    constexpr u32 SD = K2_SMEM_DESCS;         // descriptors kept in shared memory per topic; later ones spill to dpool
#ifndef GM_CPU_EMU
    extern __shared__ __align__(16) unsigned char k2_smem[];   // 64 KB: above the 48 KB static limit -> dynamic
#else
    unsigned char* k2_smem = emu::dyn_smem();
#endif
    u32 (*s_tok)[THREADS] = reinterpret_cast<u32 (*)[THREADS]>(k2_smem);                                  // tokens of this thread's topic (column = thread: conflict-free)
    u32 (*s_pend)[THREADS] = reinterpret_cast<u32 (*)[THREADS]>(k2_smem + sizeof(u32) * FAST_L * THREADS);   // parked '+' child per depth
    uint2 (*s_desc)[THREADS] = reinterpret_cast<uint2 (*)[THREADS]>(k2_smem + 2 * sizeof(u32) * FAST_L * THREADS);   // matched value sets (ref, cnt)
    const u32 tid = threadIdx.x, lane = tid & 31;
    const u32 lt = lanemask_lt();
    const u32 nthreads = gridDim.x * THREADS;
    const u32 gtid = blockIdx.x * THREADS + tid;
    const TrieView& tv = p.tv;
    const u32 n_act = p.n_ptr ? min(p.n, *p.n_ptr) : p.n;
    const u32 ntiles = (n_act + 31) >> 5;
    unsigned long long sV = 0, sE = 0, sF = 0, sM = 0;
    __shared__ unsigned long long s_chunk;
    __shared__ u32 s_lock;
    const u32 chunk = p.tile_chunk;
    if (chunk > 1) {
        if (tid == 0) { s_chunk = 0ull; s_lock = 0u; }
        __syncthreads();
    }
    for (;;) {
        u32 tile = 0;
        if (lane == 0) tile = chunk > 1 ? next_tile_chunked(&s_chunk, &s_lock, p.tile_counter, chunk) : atomicAdd(p.tile_counter, 1u);
        tile = __shfl_sync(0xFFFFFFFFu, tile, 0);
        if (tile >= ntiles) break;

        const u32 pos = tile * 32 + lane;              // position in the locality-sorted order
        const bool in_range = pos < n_act;
        const u32 t = in_range ? p.perm[pos] : 0u;     // original topic index
        const bool rows = (p.flags & MP_SORTED_ROWS) != 0;
        const u32 m = in_range ? (rows ? __ldcs(p.meta_sorted + pos) : __ldcs(p.meta + t)) : META_INVALID;
        const bool invalid = (m & META_INVALID) != 0;
        const u32 L = m & META_NLEV_MASK;
        const u32 need = min(L, tv.max_depth);
        const bool slow_pre = in_range && !invalid && need > FAST_L;
        const bool active = in_range && !invalid && !slow_pre;
        bool defer = slow_pre;
        u32 ndesc = 0, total = 0;

        if (active) {
            {
                static_assert(FAST_L == TOK8, "the token row holds 8 levels");
                u32 w[8];
                ld256(rows ? p.tok8_sorted + static_cast<size_t>(pos) * TOK8 : p.tok8 + static_cast<size_t>(t) * TOK8, w);
#pragma unroll
                for (int l = 0; l < FAST_L; ++l) s_tok[l][tid] = w[l];
            }
            NodeRec r{0u, tv.root_plus, tv.root_hash_ref, 0u, tv.root_mask, tv.root_hash_cnt};
            if (p.trees) {                             // an extra tree of the engine: start at ITS root record
                const u32 tr = p.trees[t];
                if (tr) {
                    const u32 slot = tr < tv.n_trees ? tv.tree_slots[tr] : 0xFFFFFFFFu;
                    r = NodeRec{0u, 0u, 0u, 0u, 0u, 0u};                     // no such tree: nothing can match
                    if (slot != 0xFFFFFFFFu) { u32 s8[8]; ld256(tv.edges + slot, s8); r = NodeRec{s8[2], s8[3], s8[4], s8[5], s8[6], s8[7]}; }
                }
            }
            u32 d = 0, pmask = 0;
            bool droot = (m & META_DOLLAR) != 0;      // `$`-rule: root wildcards skipped (trie.rs:312-318)
            u32 lV = 0, lE = 0, lF = 0;
            for (;;) {
                if (STATS) { lV++; lE += d < L; }
                // '#' child matches the rest of the path and, on exhaustion, the parent (trie.rs:302-308, 321-327)
                const u32 c1 = droot ? 0u : (r.cnts & 0xFFFFu);
                const u32 c2 = (d == L) ? (r.cnts >> 16) : 0u;                       // own values (trie.rs:309-310)
                if (c1) {
                    if (c1 == CNT_BIG || ndesc >= SD + pool_rows) { defer = true; break; }
                    if (ndesc < SD) s_desc[ndesc][tid] = make_uint2(r.hash_ref, c1);
                    else dpool[static_cast<size_t>(ndesc - SD) * nthreads + gtid] = Desc{r.hash_ref, c1};
                    ++ndesc; total += c1;
                    if (STATS) lF++;
                }
                if (c2) {
                    if (c2 == CNT_BIG || ndesc >= SD + pool_rows) { defer = true; break; }
                    if (ndesc < SD) s_desc[ndesc][tid] = make_uint2(r.own_ref, c2);
                    else dpool[static_cast<size_t>(ndesc - SD) * nthreads + gtid] = Desc{r.own_ref, c2};
                    ++ndesc; total += c2;
                    if (STATS) lF++;
                }
                // ---- choose the ONE slot this thread loads next: the literal child's first probe slot, else the
                // deepest parked '+' child (its record names the slot directly).  Both kinds are 32-B edge slots with
                // the same layout, so all lanes of the warp meet again at a single 32-byte load.
                u32 idx = 0, nd = 0, kp = 0, kt = 0;
                bool probe = false;
                if (d < L) {
                    if (r.plus != 0 && !droot) { s_pend[d][tid] = r.plus; pmask |= 1u << d; }   // '+' child (trie.rs:330-334)
                    if ((r.mask & MASK_BLOOM) != 0) {
                        const u32 tk = s_tok[d][tid];
                        if (tk != TOK_UNKNOWN && (r.mask & mask_bit(tk)) &&
                            (!(r.mask & MASK_WIDE_FLAG) || cfilter_maybe(tv, r.node, tk))) {        // literal child (trie.rs:338-342)
                            probe = true; kp = r.node; kt = tk; nd = d + 1;
                            idx = edge_slot0(kp, kt, r.mask >> WTAG_SHIFT, tv.win_mask, tv.win_shift, tv.nwin_mask);
                            if (STATS) atomicAdd(p.stats + 4 + min(d, 7u), 1ull);
                        }
                    }
                }
                droot = false;
                bool done = false;
                u32 s[8];
                for (;;) {
                    if (!probe) {
                        if (pmask == 0) { done = true; break; }
                        const u32 pd = 31u - __clz(pmask);          // resume the deepest parked '+' child
                        pmask &= ~(1u << pd);
                        idx = s_pend[pd][tid] - 1u;
                        nd = pd + 1;
                    }
                    ld256(tv.edges + idx, s);
                    if (!probe) break;
                    if (STATS) atomicAdd(p.stats + 20, 1ull);
                    if (s[2] == 0) {                                 // empty slot: the literal child does not exist
                        if (STATS) atomicAdd(p.stats + 12 + min(nd - 1u, 7u), 1ull);
                        probe = false;
                        continue;
                    }
                    if (s[0] == kp && s[1] == kt) break;
                    idx = edge_next(idx, tv.win_mask);               // linear probing inside the window
                }
                if (done) break;
                r.node = s[2]; r.plus = s[3]; r.hash_ref = s[4]; r.own_ref = s[5]; r.mask = s[6]; r.cnts = s[7];
                d = nd;
            }
            if (STATS && !defer) { sV += lV; sE += lE; sF += lF; sM += total; }
        }

        // ---- publish: one contiguous list per topic inside one chunk per tile ------------------------
        const u32 nd = (active && !defer) ? ndesc : 0u;
        const u32 mine = DESC ? nd : ((active && !defer) ? total : 0u);
        u32 inc = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { u32 v = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= o) inc += v; }
        const u32 wtotal = __shfl_sync(0xFFFFFFFFu, inc, 31);
        const u32 pre = inc - mine;
        unsigned long long base = 0;
        if (lane == 0 && wtotal) base = atomicAdd(p.cursor, static_cast<unsigned long long>(wtotal));
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        const bool fits = base + wtotal <= p.cap_ids;
        if (in_range && !defer) {
            if (GATHER) {        // span (absolute in the gathered id array) + global topic index into this rank's slab on EVERY rank
                const uint2 gsp = make_uint2(fits ? static_cast<u32>(p.g_base_ids + base + pre) : 0u, mine);
                const u32 gi = p.g_sel ? p.g_sel[t] : t;
                for (u32 w = 0; w < p.g_world; ++w) { p.g_spans[w][p.g_base_topics + t] = gsp; p.g_index[w][p.g_base_topics + t] = gi; }
            } else p.spans[t] = make_uint2(fits ? static_cast<u32>(base + pre) : 0u, mine);
        }
        auto store_descs = [&](uint2* __restrict__ outd) {     // this lane's nd descriptors, contiguous from outd
            for (u32 k = 0; k < nd; ++k) {
                uint2 v;
                if (k < SD) v = s_desc[k][tid];
                else { const Desc dd = dpool[static_cast<size_t>(k - SD) * nthreads + gtid]; v = make_uint2(dd.ref, dd.cnt); }
                __stcs(outd + k, v);
            }
        };
        if (DESC) {
            if (fits && wtotal) store_descs(p.out_desc + base + pre);     // this topic's descriptors, contiguous
        } else {
            // the same descriptors, lane-major (the order of their ids in out_ids), for k_match_expand — only for a tile whose
            // ids fit, so that k_match_expand writes only inside out_ids (see plan_match)
            const u32 ni = (fits && !(p.flags & MP_DIAG_NO_PUBLISH)) ? nd : 0u;
            u32 iinc = ni;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { u32 v = __shfl_up_sync(0xFFFFFFFFu, iinc, o); if (lane >= o) iinc += v; }
            const u32 witems = __shfl_sync(0xFFFFFFFFu, iinc, 31);
            u32 ibase = 0;      // (items stay below cap_ids <= 2^32 - 1)
            if (lane == 0 && witems) ibase = static_cast<u32>(atomicAdd(p.item_cursor, static_cast<unsigned long long>(witems)));
            ibase = __shfl_sync(0xFFFFFFFFu, ibase, 0);
            if (lane == 0) p.tiles[tile] = TileRec{ibase, witems, base};
            if (ni) store_descs(p.items + ibase + (iinc - ni));
        }
        const bool deferred = in_range && defer;
        u32 db = __ballot_sync(0xFFFFFFFFu, deferred);
        if (db) {
            u32 sb = 0;
            if (lane == 0) sb = atomicAdd(p.slow_count, static_cast<u32>(__popc(db)));
            sb = __shfl_sync(0xFFFFFFFFu, sb, 0);
            if (deferred) p.slow_list[sb + __popc(db & lt)] = t;
        }
    }
    if (STATS) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            sV += __shfl_xor_sync(0xFFFFFFFFu, sV, o); sE += __shfl_xor_sync(0xFFFFFFFFu, sE, o);
            sF += __shfl_xor_sync(0xFFFFFFFFu, sF, o); sM += __shfl_xor_sync(0xFFFFFFFFu, sM, o);
        }
        if (lane == 0) { atomicAdd(p.stats + 0, sV); atomicAdd(p.stats + 1, sE); atomicAdd(p.stats + 2, sF); atomicAdd(p.stats + 3, sM); }
    }
}

// K2b: the ids of k_match_fast's tiles.  One warp per tile record; the tile's value sets (ref, cnt) are in id order and
// are taken 32 at a time: warp scan of cnt, then every lane finds the set of its flat index (warp_run_owner) and copies one
// id, so each 32-id step is one contiguous 128-byte run of out_ids.  GATHER: the ids go into the gathered array of every
// rank in g_ids (push form: the own block only).
template <bool GATHER>
__global__ void __launch_bounds__(256)
k_match_expand(MatchParams p) {
    const u32 lane = threadIdx.x & 31;
    const u32 gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    const u32 n_act = p.n_ptr ? min(p.n, *p.n_ptr) : p.n;
    const u32 ntiles = (n_act + 31) >> 5;
    for (u32 tile = gwarp; tile < ntiles; tile += nwarps) {
        const TileRec rec = p.tiles[tile];
        unsigned long long at = (GATHER ? p.g_base_ids : 0ull) + rec.id_base;
        for (u32 i0 = 0; i0 < rec.n_items; i0 += 32) {
            const u32 i = i0 + lane;
            const uint2 d = i < rec.n_items ? __ldcs(p.items + rec.item_base + i) : make_uint2(0u, 0u);
            u32 sc = d.y;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { u32 v = __shfl_up_sync(0xFFFFFFFFu, sc, o); if (lane >= o) sc += v; }
            const u32 tot = __shfl_sync(0xFFFFFFFFu, sc, 31);
            const u32 exc = sc - d.y;
            // with owner o: source index = e + (ref_o - exc_o); a one-value set has e == exc_o, so its value ref_o is that too
            const u32 gamma = d.x - exc;
            const u32 single = __ballot_sync(0xFFFFFFFFu, d.y == 1u);
            for (u32 e0 = 0; e0 < tot; e0 += 32) {
                const u32 e = e0 + lane;
                const u32 o = warp_run_owner(exc, e);
                const u32 src = e + __shfl_sync(0xFFFFFFFFu, gamma, o);
                if (e < tot) {
                    const u32 val = ((single >> o) & 1u) ? src : p.tv.values[src];
                    if (GATHER) { for (u32 w = 0; w < p.g_world; ++w) p.g_ids[w][at + e] = val; }   // posted stores, NVLink for the peers
                    else __stcs(p.out_ids + at + e, val);                                          // streaming store: written once
                }
            }
            at += tot;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K3: one warp per deferred topic; pass 0 counts, pass 1 writes.  The frontier stack lives in global
// scratch (gstack, `stack_cap` items per warp: 32*(max_depth+2)+64 bounds the LIFO walk).
// In STATS mode the counters of a deferred topic are taken here (the fast path's partial counts of
// topics it later deferred are subtracted by never being added: see `stats_defer` below).
template <bool STATS, bool DESC, bool GATHER = false>
__global__ void __launch_bounds__(256)
k_match_slow(MatchParams p, u64* __restrict__ gstack, u32 stack_cap) {
    auto put = [&](unsigned long long at, u32 v) {       // one result id: local array, or every rank's gathered array
        if (GATHER) { for (u32 w = 0; w < p.g_world; ++w) p.g_ids[w][p.g_base_ids + at] = v; }
        else p.out_ids[at] = v;
    };
    const u32 lane = threadIdx.x & 31;
    const u32 lt = lanemask_lt();
    const u32 gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const u32 nwarps = (gridDim.x * blockDim.x) >> 5;
    const TrieView& tv = p.tv;
    u64* stack = gstack + static_cast<size_t>(gwarp) * stack_cap;
    const u32 nslow = *p.slow_count;
    unsigned long long sV = 0, sE = 0, sF = 0, sM = 0;

    for (u32 si = gwarp; si < nslow; si += nwarps) {
        const u32 t = p.slow_list[si];
        const u32 m = p.meta[t];
        const u32 L = m & META_NLEV_MASK;
        const bool dollar = (m & META_DOLLAR) != 0;
        unsigned long long base = 0;
        unsigned long long count = 0;
        bool fits = true, bad_any = false;
        for (int pass = 0; pass < 2; ++pass) {
            u32 stack_n = 0;
            unsigned long long written = 0;
            bool bad = false;
            auto consume = [&](bool hit, u32 d, const NodeRec& r, bool dollar_root) {
                const u32 c1 = (hit && !dollar_root) ? (r.cnts & 0xFFFFu) : 0u;
                const u32 c2 = (hit && d == L) ? (r.cnts >> 16) : 0u;
                u64 itA = 0, itB = 0;
                bool pA = false, pB = false;
                if (hit && d < L) {
                    const u32 plus_idx = r.plus;
                    if (plus_idx != 0 && !dollar_root) { pA = true; itA = make_item(0, d + 1, KIND_PLUS, plus_idx); }
                    if ((r.mask & MASK_BLOOM) != 0 && d < p.tok_levels) {
                        u32 tk = d < TOK8 ? p.tok8[static_cast<size_t>(t) * TOK8 + d] : p.tok[static_cast<size_t>(d) * p.n + t];
                        if (tk != TOK_UNKNOWN && (r.mask & mask_bit(tk)) && (!(r.mask & MASK_WIDE_FLAG) || cfilter_maybe(tv, r.node, tk))) {
                            pB = true; itB = make_item(0, d + 1, KIND_PROBE, r.node, r.mask >> WTAG_SHIFT);
                        }
                    }
                }
                if (STATS && pass == 0) { sV += hit; sE += (hit && d < L); }
#pragma unroll
                for (int round = 0; round < 2; ++round) {
                    const u32 cn = round == 0 ? c1 : c2;
                    const u32 ref = round == 0 ? r.hash_ref : r.own_ref;
                    if (STATS && pass == 0) sF += (cn != 0);
                    if (DESC) {                 // one (ref, cnt16) descriptor per matched value set; CNT_BIG sets resolve through `ranges` on the host
                        const u32 bd = __ballot_sync(0xFFFFFFFFu, cn != 0);
                        if (pass == 1 && cn != 0) p.out_desc[base + written + __popc(bd & lt)] = make_uint2(ref, cn);
                        written += __popc(bd);
                        if (STATS && pass == 0 && cn != 0) sM += cn == CNT_BIG ? tv.ranges[ref].cnt : cn;
                        continue;
                    }
                    u32 b = __ballot_sync(0xFFFFFFFFu, cn == 1);
                    if (pass == 1 && cn == 1) put(base + written + __popc(b & lt), ref);
                    written += __popc(b);
                    u32 rb = __ballot_sync(0xFFFFFFFFu, cn > 1);
                    while (rb) {     // warp-cooperative copy of one value set at a time
                        int leader = __ffs(rb) - 1;
                        rb &= rb - 1;
                        u32 rr = __shfl_sync(0xFFFFFFFFu, ref, leader);
                        u32 rc = __shfl_sync(0xFFFFFFFFu, cn, leader);
                        u32 off = rr;
                        if (rc == CNT_BIG) { Range rg = tv.ranges[rr]; off = rg.off; rc = rg.cnt; }
                        if (pass == 1)
                            for (u32 i = lane; i < rc; i += 32) put(base + written + i, tv.values[off + i]);
                        written += rc;
                    }
                }
#pragma unroll
                for (int round = 0; round < 2; ++round) {
                    const bool push = round == 0 ? pA : pB;
                    u32 b = __ballot_sync(0xFFFFFFFFu, push);
                    if (b) {
                        u32 tot = __popc(b);
                        if (stack_n + tot <= stack_cap) {
                            if (push) stack[stack_n + __popc(b & lt)] = round == 0 ? itA : itB;
                            stack_n += tot;
                        } else bad = true;
                    }
                }
                __syncwarp();
            };
            {
                NodeRec r{0u, tv.root_plus, tv.root_hash_ref, 0u, tv.root_mask, tv.root_hash_cnt};
                const u32 tr = p.trees ? p.trees[t] : 0u;
                if (tr) {
                    const u32 slot = tr < tv.n_trees ? tv.tree_slots[tr] : 0xFFFFFFFFu;
                    r = NodeRec{0u, 0u, 0u, 0u, 0u, 0u};
                    if (slot != 0xFFFFFFFFu) { u32 s8[8]; ld256(tv.edges + slot, s8); r = NodeRec{s8[2], s8[3], s8[4], s8[5], s8[6], s8[7]}; }
                }
                consume(lane == 0, 0u, r, dollar);
            }
            while (stack_n) {
                const u32 take = min(stack_n, 32u);
                const bool have = lane < take;
                __threadfence_block();
                u64 it = have ? stack[stack_n - 1 - lane] : 0ull;
                stack_n -= take;
                __syncwarp();
                const u32 hi = static_cast<u32>(it >> 32), arg = static_cast<u32>(it);
                const u32 d = (hi >> 5) & 0xFFFFu, kind = (hi >> 21) & 1u;
                NodeRec r{};
                bool hit = false;
                if (have) {
                    u32 tk = 0u;
                    if (kind == KIND_PROBE) tk = (d - 1) < TOK8 ? p.tok8[static_cast<size_t>(t) * TOK8 + (d - 1)] : p.tok[static_cast<size_t>(d - 1) * p.n + t];
                    hit = load_record(tv, kind, arg, tk, ((hi >> 22) & 0xFFu) << WTAG_SHIFT, r);
                }
                consume(hit, d, r, false);
            }
            if (pass == 0) {
                count = written;
                if (STATS && !DESC) sM += (lane == 0) ? count : 0;
                if (lane == 0 && count) base = atomicAdd(p.cursor, count);
                base = __shfl_sync(0xFFFFFFFFu, base, 0);
                bad_any = bad;
                fits = !bad && (base + count <= p.cap_ids) && count <= 0xFFFFFFFFull;
                if (!fits) break;
            }
        }
        if (lane == 0) {
            // a frontier-stack overflow cannot happen within the documented bound; if it ever did, fail the topic loudly
            // instead of aliasing another topic's list (ADVICE r1)
            uint2 sp = make_uint2(fits ? static_cast<u32>(base) : 0u, static_cast<u32>(count));
            if (bad_any) { sp = make_uint2(0u, 0u); p.status[t] = -8; }   // GM_ERR_INTERNAL
            if (GATHER) {
                if (fits && !bad_any) sp.x = static_cast<u32>(p.g_base_ids + base);
                const u32 gi = p.g_sel ? p.g_sel[t] : t;
                for (u32 w = 0; w < p.g_world; ++w) { p.g_spans[w][p.g_base_topics + t] = sp; p.g_index[w][p.g_base_topics + t] = gi; }
            } else p.spans[t] = sp;
        }
    }
    if (STATS) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            sV += __shfl_xor_sync(0xFFFFFFFFu, sV, o); sE += __shfl_xor_sync(0xFFFFFFFFu, sE, o);
            sF += __shfl_xor_sync(0xFFFFFFFFu, sF, o); sM += __shfl_xor_sync(0xFFFFFFFFu, sM, o);
        }
        if (lane == 0) { atomicAdd(p.stats + 0, sV); atomicAdd(p.stats + 1, sE); atomicAdd(p.stats + 2, sF); atomicAdd(p.stats + 3, sM); }
    }
}

// ------------------------------------------------------------------------------------------------
// Flush: scatter patches (EdgeSlot / DictSlot / RKid / REdge: 32 B, Range: 8 B, retained value words: 4 B) into a device table.
template <class T>
__global__ void k_apply_patches(T* __restrict__ table, const u32* __restrict__ idx, const T* __restrict__ data, u32 n) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    table[idx[i]] = data[i];
}

}  // namespace gm
