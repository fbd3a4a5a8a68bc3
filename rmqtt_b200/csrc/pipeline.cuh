// How the match and retained-lookup kernels are driven: the control blocks, the scratch plan, the launch sequences, the
// table views, the fused-gather block layout and what a flush ships.  engine.cu runs these on the GPU; the CPU emulation
// (tests/native/emu, -DGM_CPU_EMU) runs the same code over host memory, so a mistake here fails the CPU tier too.
// Stream waits, memsets, completion events, graph capture and the capacity protocol stay with the engine.
#pragma once
#include <algorithm>
#include <cstddef>

#include "../../include/gpumqtt.h"
#include "host_trie.h"
#include "kernels.cuh"
#include "retain_kernels.cuh"
#include "retain_tree.h"

namespace gm {

// ---- control blocks ----------------------------------------------------------------------------------------------------
// match control block, zeroed before every match (a pipelined host call keeps `cursor` across its chunks and clears the rest,
// item_cursor included: every chunk has its own item array)
struct Ctrl { unsigned long long cursor; unsigned long long item_cursor; unsigned long long stats[24]; u32 slow_count; u32 tile_counter; };

// Retained-lookup control block.  counts[(depth + 3) * RQ] (tasks queued per round and queue slice; round 0 = k_retain_init)
// and claim[depth + 3] (the task hand-out of every round) follow it in the same allocation.
struct RCtl {
    unsigned long long grand; unsigned long long stats[2]; u32 err; u32 pad; u32 n_desc[RQ]; u32 counts[RQ];
    static size_t bytes(u32 depth) { return sizeof(RCtl) + static_cast<size_t>(depth + 3) * RQ * sizeof(u32) + static_cast<size_t>(depth + 3) * sizeof(u32); }
    u32* round_counts(u32 lvl) { return counts + static_cast<size_t>(lvl) * RQ; }
    u32* claim(u32 depth, u32 lvl) { return counts + static_cast<size_t>(depth + 3) * RQ + lvl; }
};

// fast-path geometry (see DESIGN.md): one topic per thread, 512 threads per CTA, 3 CTAs per SM (64 KB of shared memory each)
constexpr int K2_FAST_L = 8;       // levels staged in shared memory; deeper topics take the deferred kernel
constexpr int K2_THREADS = 512;
constexpr int K2_CTAS_PER_SM = 3;
constexpr u32 K2_POOL_ROWS = 24;   // matched value sets per topic beyond the 8 held in shared memory, before the topic is deferred
constexpr size_t K2_SMEM = k2_smem_bytes<K2_FAST_L, K2_THREADS>();

// the k_match_fast / k_match_slow instantiation of a launch (the fused gather has no instrumented or descriptor form)
inline auto k2_kernel(bool stats, bool desc, bool gather) {
    return gather ? k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, false, false, true>
         : stats  ? (desc ? k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, true, true> : k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, true, false>)
                  : (desc ? k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, false, true> : k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, false, false>);
}
inline auto k3_kernel(bool stats, bool desc, bool gather) {
    return gather ? k_match_slow<false, false, true>
         : stats  ? (desc ? k_match_slow<true, true> : k_match_slow<true, false>) : (desc ? k_match_slow<false, true> : k_match_slow<false, false>);
}

// ---- the scratch plan --------------------------------------------------------------------------------------------------
// 2^(site_bits + sub_bits) locality buckets; k2_ctas: k_match_fast CTAs per SM (outside 1 .. K2_CTAS_PER_SM: K2_CTAS_PER_SM)
struct MatchKnobs { u32 site_bits = 14, sub_bits = 0; bool sorted_rows = true; int k2_ctas = 0; u32 diag_flags = 0; u32 tile_chunk = 1; bool tok_bulk = true; u32 pool_rows = K2_POOL_ROWS; };

inline size_t tok_bytes(u32 tok_levels, u32 n) { return tok_levels > TOK8 ? static_cast<size_t>(tok_levels) * n * sizeof(u32) : 256; }   // levels >= 8 only

// Sizes (bytes) of every scratch array of one match launch, and its grids.  `small`: the small-graph form, launched for a
// capacity of n rows while the real batch size is read from `hdr` at run time; its fast and deferred grids are capped to n rows.
struct MatchPlan {
    u32 n, tok_levels, nbuckets, stack_cap, pool_rows;
    int tok_grid, scatter_grid, k2_grid, expand_grid, k3_blocks;
    size_t tok, tok8, meta, slow, ctrl, sort, hist, gstack, gpool;
};
inline MatchPlan plan_match(u32 n, u32 max_depth, const MatchKnobs& kn, int num_sms, bool small) {
    MatchPlan p{};
    p.n = n;
    p.tok_levels = std::max<u32>(1u, max_depth);
    p.nbuckets = 1u << (kn.site_bits + kn.sub_bits);
    p.stack_cap = 32u * (max_depth + 2u) + 64u;
    p.pool_rows = kn.pool_rows;
    const int k2_ctas = (kn.k2_ctas >= 1 && kn.k2_ctas <= K2_CTAS_PER_SM) ? kn.k2_ctas : K2_CTAS_PER_SM;
    p.tok_grid = static_cast<int>((n + TOK_THREADS - 1) / TOK_THREADS);
    p.scatter_grid = static_cast<int>((n + 255) / 256);
    p.k2_grid = small ? std::max(1, std::min<int>(num_sms * k2_ctas, (n + K2_THREADS - 1) / K2_THREADS)) : num_sms * k2_ctas;
    p.expand_grid = small ? std::max(1, std::min<int>(num_sms * 8, (n + 255) / 256)) : num_sms * 8;   // 8 warps of 256 threads, one tile each
    p.k3_blocks = small ? std::max(1, std::min<int>(num_sms, (n + 7) / 8)) : num_sms * 4;
    p.tok = tok_bytes(p.tok_levels, n); p.tok8 = static_cast<size_t>(n) * TOK8 * sizeof(u32);
    p.meta = p.slow = n * sizeof(u32); p.ctrl = sizeof(Ctrl);
    // carved in launch_match: the locality order and sorted rows, then k_match_fast's tile records and value sets (ids mode).
    // Only a tile whose ids fit stores its value sets, and a topic with more than K2_SMEM_DESCS + K2_POOL_ROWS (32) of them
    // is deferred: at most 32 per row, whatever the output's capacity.  (Storing them only for tiles that fit also keeps
    // k_match_expand inside the output: every set has at least one id, and those tiles' ids are disjoint ranges below cap_ids.)
    p.sort = static_cast<size_t>(n) * 11 * sizeof(u32) + 64 + static_cast<size_t>((n + 31) / 32) * sizeof(TileRec) + 32ull * n * sizeof(uint2);
    p.hist = 2 * static_cast<size_t>(p.nbuckets) * sizeof(u32);     // counts[nbuckets] | cursor[nbuckets]
    p.gstack = static_cast<size_t>(num_sms) * 4 * 8 * p.stack_cap * sizeof(u64);
    p.gpool = static_cast<size_t>(num_sms) * k2_ctas * K2_THREADS * p.pool_rows * sizeof(Desc);
    return p;
}

struct RetainPlan {
    u32 nq, depth, tok_levels, slice_items, slice_desc;
    int tok_grid, init_grid, round_grid, expand_grid;
    size_t tok, tok8, meta, rq, ctl, front, descs;   // bytes; `front`: each of the two frontier queues; rq: qtotal | qbase | qcur [nq] each
};
// cap_items / cap_desc: totals over the RQ slices of each queue
inline RetainPlan plan_retain(u32 nq, u32 depth, u32 cap_items, u32 cap_desc, int num_sms) {
    RetainPlan p{};
    p.nq = nq; p.depth = depth;
    p.tok_levels = depth + 2;                        // the walk reads filter levels pos and pos+1 with pos <= tree depth
    p.slice_items = std::max<u32>(1u, cap_items / RQ); p.slice_desc = std::max<u32>(1u, cap_desc / RQ);
    p.tok_grid = static_cast<int>((nq + TOK_THREADS - 1) / TOK_THREADS);
    p.init_grid = static_cast<int>((nq + 255) / 256);
    p.round_grid = num_sms * GM_RETAIN_CTAS;         // exactly the resident CTAs (launch bound of k_retain_round): tasks are claimed dynamically
    p.expand_grid = num_sms * 8;
    p.tok = tok_bytes(p.tok_levels, nq); p.tok8 = static_cast<size_t>(nq) * TOK8 * sizeof(u32); p.meta = nq * sizeof(u32);
    p.rq = static_cast<size_t>(nq) * 3 * sizeof(u32); p.ctl = RCtl::bytes(depth);
    p.front = static_cast<size_t>(p.slice_items) * RQ * sizeof(RTask); p.descs = static_cast<size_t>(p.slice_desc) * RQ * sizeof(RDesc);
    return p;
}

// ---- the fused-gather block (comm.cuh): one per rank, holding every rank's slab -----------------------------------------
struct GatherLayout {
    static constexpr size_t off_ids = 256;      // the block starts with a 256-byte header {world, slab_topics, slab_ids}
    u32 world = 0; u64 slab_topics = 0, slab_ids = 0;
    size_t off_spans = 0, off_index = 0, off_counts = 0, off_flags = 0, bytes = 0;
};
inline GatherLayout gather_layout(u32 world, u64 slab_topics, u64 slab_ids) {
    GatherLayout g;
    g.world = world; g.slab_topics = (slab_topics + 3) & ~u64(3); g.slab_ids = (slab_ids + 3) & ~u64(3);       // every slab starts on a 16-byte boundary
    const size_t a = 256;
    g.off_spans = (GatherLayout::off_ids + static_cast<size_t>(world) * g.slab_ids * 4 + a - 1) / a * a;
    g.off_index = g.off_spans + static_cast<size_t>(world) * g.slab_topics * 8;
    g.off_counts = (g.off_index + static_cast<size_t>(world) * g.slab_topics * 4 + a - 1) / a * a;
    g.off_flags = g.off_counts + static_cast<size_t>(world) * 16;
    g.bytes = g.off_flags + 256;
    return g;
}
// where a rank's fused-gather match publishes: `direct`, into every rank's block itself; else into its own block only, and
// k_gather_push copies the slab to the peers
struct GatherTarget { const GatherLayout* layout; char* const* blocks; u32 rank; bool direct; };

// ---- the launch sequences ----------------------------------------------------------------------------------------------
struct MatchScratch { u32 *tok, *tok8, *meta, *slow, *sort, *hist; Ctrl* ctrl; u64* gstack; Desc* gpool; };

// one batch: where its text comes from and where the results go
struct MatchIO {
    const void* blob = nullptr; u64 blob_bytes = 0, readable_bytes = 0;   // readable: bytes the bulk tokeniser may read (at least blob_bytes)
    const u32* offs = nullptr;
    const u32* sel = nullptr;                    // optional selection: row t matches entry sel[t] of the packed batch
    u64 n = 0;
    const u32* hdr = nullptr;                    // small-graph form: {n, blob_bytes} in memory, read at run time; n is then the capacity
    const u32* trees = nullptr;                  // optional: the tree every row is matched against
    gm_span* spans = nullptr; void* out = nullptr; u64 cap = 0;   // out: ids, or descriptors (uint2) with `desc`
    int32_t* status = nullptr;
    bool stats = false, desc = false;            // the instrumented instantiations (V / E / F / M counters); descriptor mode
    const GatherTarget* gather = nullptr;        // the fused-gather instantiations
};

struct NoHook { void operator()(int) const {} };

// k_tokenize -> k_bucket_scan -> k_bucket_scatter -> k_match_fast -> k_match_expand (ids only) -> k_match_slow.  `at(k)` runs
// before the tokeniser (0), after the locality pass (1), after the fast kernel and the expansion (2) and after the deferred
// kernel (3).
template <class Hook = NoHook>
inline void launch_match(const MatchPlan& p, const MatchScratch& m, const MatchIO& io, const MatchKnobs& kn, const TrieView& tv, cudaStream_t s, Hook at = {}) {
    const u32 n = p.n;
    u32* bkey = m.sort;            // sort: bkey[n] | perm[n] | meta_sorted[n] | padding to 32 bytes | tok8_sorted[n][8] | tiles | items
    u32* perm = bkey + n;
    u32* meta_sorted = perm + n;
    u32* tok8_sorted = meta_sorted + n + ((8 - (3 * static_cast<size_t>(n)) % 8) % 8);   // 32-byte aligned rows
    TileRec* tiles = reinterpret_cast<TileRec*>(tok8_sorted + static_cast<size_t>(n) * TOK8);  // ... then tile records | value sets
    uint2* items = reinterpret_cast<uint2*>(tiles + (n + 31) / 32);
    u32* bcursor = m.hist + p.nbuckets;
    at(0);
    auto k1 = kn.tok_bulk ? k_tokenize<true> : k_tokenize<false>;
    GM_LAUNCH(k1, p.tok_grid, TOK_THREADS, 0, s, static_cast<const u8*>(io.blob), static_cast<u32>(io.blob_bytes), static_cast<u32>(std::max<u64>(io.blob_bytes, io.readable_bytes)),
              io.offs, io.sel, n, io.hdr, tv, p.tok_levels, m.tok8, m.tok, m.meta, io.status, bkey, m.hist, kn.site_bits, kn.sub_bits);
    GM_LAUNCH(k_bucket_scan, 1, 1024, 0, s, m.hist, bcursor, p.nbuckets);
    GM_LAUNCH(k_bucket_scatter, p.scatter_grid, 256, 0, s, bkey, bcursor, n, io.hdr, perm, m.tok8, m.meta, kn.sorted_rows ? tok8_sorted : nullptr, meta_sorted);
    at(1);
    MatchParams mp{};
    mp.tv = tv; mp.tok8 = m.tok8; mp.tok = m.tok; mp.meta = m.meta; mp.n = n; mp.n_ptr = io.hdr; mp.tok_levels = p.tok_levels;
    mp.spans = reinterpret_cast<uint2*>(io.spans); mp.out_ids = static_cast<u32*>(io.out); mp.out_desc = static_cast<uint2*>(io.out); mp.cap_ids = io.cap;
    mp.status = io.status;
    mp.items = items; mp.tiles = tiles; mp.item_cursor = &m.ctrl->item_cursor;
    mp.trees = io.trees;
    mp.cursor = &m.ctrl->cursor; mp.slow_list = m.slow; mp.slow_count = &m.ctrl->slow_count;
    mp.tile_counter = &m.ctrl->tile_counter; mp.stats = m.ctrl->stats;
    mp.perm = perm; mp.tok8_sorted = tok8_sorted; mp.meta_sorted = meta_sorted;
    mp.flags = (kn.sorted_rows ? MP_SORTED_ROWS : 0u) | kn.diag_flags;
    mp.tile_chunk = kn.tile_chunk;
    if (const GatherTarget* g = io.gather) {
        const GatherLayout& L = *g->layout;
        mp.g_base_topics = static_cast<u32>(g->rank * L.slab_topics); mp.g_base_ids = g->rank * L.slab_ids; mp.g_sel = io.sel;
        mp.g_world = g->direct ? L.world : 1;
        for (u32 w = 0; w < mp.g_world; ++w) {
            char* b = g->blocks[g->direct ? w : g->rank];
            mp.g_ids[w] = reinterpret_cast<u32*>(b + GatherLayout::off_ids); mp.g_spans[w] = reinterpret_cast<uint2*>(b + L.off_spans);
            mp.g_index[w] = reinterpret_cast<u32*>(b + L.off_index);
        }
    }
    const bool gather = io.gather != nullptr;
    auto k2 = k2_kernel(io.stats, io.desc, gather);
    GM_LAUNCH(k2, p.k2_grid, K2_THREADS, K2_SMEM, s, mp, m.gpool, p.pool_rows);
    if (!io.desc) {
        auto kx = gather ? k_match_expand<true> : k_match_expand<false>;
        GM_LAUNCH(kx, p.expand_grid, 256, 0, s, mp);
    }
    at(2);
    auto k3 = k3_kernel(io.stats, io.desc, gather);
    GM_LAUNCH(k3, p.k3_blocks, 256, 0, s, mp, m.gstack, p.stack_cap);
    at(3);
}

struct RetainScratch { u32 *tok, *tok8, *meta, *rq; RCtl* ctl; RTask* front[2]; RDesc* descs; };

// k_tokenize -> k_retain_init -> k_retain_round x (depth + 1) -> k_retain_scan -> k_retain_expand.  `at(k)` runs before the
// tokeniser (0), after it (1), after the last round (2) and after the expansion (3).
template <class Hook = NoHook>
inline void launch_retain(const RetainPlan& p, const RetainScratch& r, const TrieView& tv, const RetainView& rv, const void* blob, u64 blob_bytes, const u32* offs,
                          gm_span* spans, u32* ids, u64 cap_ids, int32_t* status, bool stats, cudaStream_t s, Hook at = {}) {
    const u32 nq = p.nq, depth = p.depth;
    u32* qtotal = r.rq;
    u32* qbase = qtotal + nq;
    u32* qcur = qbase + nq;
    at(0);
    GM_LAUNCH(k_tokenize<false>, p.tok_grid, TOK_THREADS, 0, s, static_cast<const u8*>(blob), static_cast<u32>(blob_bytes), static_cast<u32>(blob_bytes), offs, nullptr, nq, nullptr, tv,
              p.tok_levels, r.tok8, r.tok, r.meta, status, nullptr, nullptr, 0u, 0u);
    at(1);
    RetainParams rp{};
    rp.v = rv; rp.qtok8 = r.tok8; rp.qtok = r.tok; rp.qmeta = r.meta; rp.nq = nq; rp.tok_levels = p.tok_levels;
    rp.descs = r.descs; rp.n_desc = r.ctl->n_desc; rp.cap_items = p.slice_items; rp.cap_desc = p.slice_desc;
    rp.qtotal = qtotal; rp.err = &r.ctl->err;
    rp.stats = r.ctl->stats;
    // round 0 follows every filter's literal prefix; every later round expands the wildcard tasks the round before
    // queued.  A task descends at least one tree level, so depth + 1 rounds drain every queue (late rounds find
    // theirs empty and return at once).
    auto kri = stats ? k_retain_init<true> : k_retain_init<false>;
    auto krr = stats ? k_retain_round<true> : k_retain_round<false>;
    GM_LAUNCH(kri, p.init_grid, 256, 0, s, rp, r.front[0], r.ctl->round_counts(0));
    for (u32 lvl = 0; lvl <= depth; ++lvl)
        GM_LAUNCH(krr, p.round_grid, 256, 0, s, rp, r.front[lvl & 1], r.ctl->round_counts(lvl), r.front[(lvl + 1) & 1], r.ctl->round_counts(lvl + 1), r.ctl->claim(depth, lvl));
    at(2);
    GM_LAUNCH(k_retain_scan, 1, 1024, 0, s, qtotal, nq, qbase, reinterpret_cast<uint2*>(spans), &r.ctl->grand);
    GM_LAUNCH(k_retain_expand, p.expand_grid, 256, 0, s, r.descs, r.ctl->n_desc, p.slice_desc, rv.vals, qbase, qcur, ids, cap_ids);
    at(3);
}

// tokenise only (gm_tokenize_batch): tokens and meta words of every level, no locality pass
inline void launch_tokenize(bool bulk, const void* blob, u64 blob_bytes, const u32* offs, u32 n, const TrieView& tv, u32 tok_levels, u32* tok8, u32* tok, u32* meta,
                            int32_t* status, cudaStream_t s) {
    auto k = bulk ? k_tokenize<true> : k_tokenize<false>;
    GM_LAUNCH(k, (n + TOK_THREADS - 1) / TOK_THREADS, TOK_THREADS, 0, s, static_cast<const u8*>(blob), static_cast<u32>(blob_bytes), static_cast<u32>((blob_bytes + 15) & ~u64(15)),
              offs, nullptr, n, nullptr, tv, tok_levels, tok8, tok, meta, status, nullptr, nullptr, 0u, 0u);
}

// ---- the views the kernels get: table geometry from the host mirror, table pointers from the caller ----------------------
inline TrieView trie_view(const HostTrie& t, const EdgeSlot* edges, const Range* ranges, const u32* values, const DictSlot* dict, const u8* pool, const u32* cfilter,
                          const u32* tree_slots) {
    TrieView v{};
    v.edges = edges; v.ranges = ranges; v.values = values; v.dict = dict; v.pool = pool;
    v.cfilter = cfilter; v.cfilter_mask = static_cast<u32>(t.cfilter.size() - 1);
    v.edge_mask = static_cast<u32>(t.edges.size() - 1);
    v.win_mask = t.win_mask(); v.win_shift = t.win_shift(); v.nwin_mask = t.nwin_mask();
    v.dict_mask = static_cast<u32>(t.dict.size() - 1);
    v.root_plus = t.root_plus; v.root_hash_ref = t.root_hash_ref; v.root_hash_cnt = t.root_hash_cnt; v.root_mask = t.root_mask;
    v.max_depth = t.max_depth;
    v.tree_slots = tree_slots; v.n_trees = tree_slots ? static_cast<u32>(t.tree_slots.size()) : 0u;   // no tree slots shipped yet: no extra trees
    return v;
}

inline RetainView retain_view(const RetainTreeHost& t, const RKid* kids, const REdge* edges, const u32* vals) {
    RetainView v{};
    v.kids = kids; v.edges = edges; v.vals = vals;
    v.edge_mask = static_cast<u32>(t.redges.size() - 1);
    if (!t.rnodes.empty()) { v.root_first_kid = t.rnodes[0].first_kid; v.root_nk_flags = t.rnodes[0].nkids | (t.rnodes[0].flags << 28); }
    v.root_plain_kids = t.root_plain_kids; v.root_plain_val_hi = t.root_plain_val_hi; v.max_depth = t.max_depth;
    v.n_kids = static_cast<u32>(t.rkids.size());
    return v;
}

// ---- what a flush ships --------------------------------------------------------------------------------------------------
// Hash tables (edges, dict, retained edges): the whole table into a fresh buffer after a re-hash, on its first shipment or when
// more than an eighth of it changed; otherwise only its dirty slots.
inline bool ship_table_whole(bool full, size_t shipped_slots, size_t slots, size_t n_dirty) { return full || shipped_slots != slots || n_dirty * 8 > slots; }

// Append-only arrays (ranges, values, pool, retained child blocks / values): a fresh buffer on the first shipment, after the
// content was rebuilt (shipped reset to 0) or when the array outgrew its buffer; otherwise the new tail is appended in place.
inline bool ship_appendable_fresh(size_t shipped, size_t bytes, bool have_buffer, size_t buffer_bytes) { return (shipped == 0 && (bytes > 0 || !have_buffer)) || bytes > buffer_bytes; }
inline size_t appendable_room(size_t bytes) { return std::max(bytes * 2, size_t(4096)); }   // a fresh appendable buffer: room to append as much again

// bytes of a fresh buffer for `bytes` of content
inline size_t fresh_bytes(size_t bytes, size_t min_bytes, size_t slack_bytes) { return std::max<size_t>(std::max(bytes + slack_bytes, min_bytes), 256); }
// a retained tree shipped whole (after a (re)flatten) gets room for in-place appends
inline size_t retained_kids_slack(size_t n_kids) { return (n_kids / 4 + 1024) * sizeof(RKid); }
constexpr size_t RETAINED_VALS_SLACK = 4096;

}  // namespace gm
