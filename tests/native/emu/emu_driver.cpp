// TEST INFRASTRUCTURE: the match and retained-lookup pipelines of engine.cu (enqueue_match / enqueue_retain) over HOST
// memory, with the REAL kernel sources (kernels.cuh, retain_kernels.cuh, relations.cuh compiled with -DGM_CPU_EMU) run
// by the CPU emulation in cuda_runtime.h.  Exposed as a small C interface for tests/test_emu_kernels.py, which compares
// the results with the oracle.  Build (tests/test_emu_kernels.py does it):
//   g++ -O1 -g -std=c++17 -DGM_CPU_EMU -Itests/native/emu -Irmqtt_b200/csrc -shared -fPIC tests/native/emu/emu_driver.cpp \
//       rmqtt_b200/csrc/host_trie.cpp rmqtt_b200/csrc/retain_tree.cpp -o <out>.so     (+ -fsanitize=address,undefined for the ASan run)
#include <cuda_runtime.h>      // the emulation (this directory is first on the include path)

#include <cstring>
#include <vector>

#include "../../../include/gpumqtt.h"
#include "comm.cuh"
#include "host_trie.h"
#include "kernels.cuh"
#include "relations.cuh"
#include "retain_kernels.cuh"
#include "retain_tree.h"

using namespace gm;

namespace {

struct Ctrl { unsigned long long cursor; unsigned long long stats[24]; u32 slow_count; u32 tile_counter; };   // engine.cu's control block

constexpr int K2_FAST_L = 8, K2_THREADS = 512, K2_CTAS_PER_SM = 3;
constexpr u32 EMU_SMS = 2;               // the emulated part has two SMs: several CTAs per kernel, dynamic tile hand-out exercised

// A "device copy" of one table, maintained ONLY by what gm_engine::flush_impl would ship (engine.cu upload_table /
// upload_appendable / stage_patches): whole arrays after a re-hash or for the first shipment, appended tails, and the slots the
// host mirror listed as dirty.  A slot the mirror changed without listing it stays stale here — and shows up as a wrong match.
template <class T> struct ImgBuf {
    std::vector<T> v;                    // v.size() plays the role of DevBuf::cap (elements)
    size_t up = 0;                       // shipped up to here (appendable arrays) / shipped size (tables)
    bool have = false;
    template <class H> void fresh(const H& host, size_t min_elems) {
        v.assign(std::max(std::max(host.size(), min_elems), size_t(8)), T{});
        std::memset(static_cast<void*>(v.data()), 0xCD, v.size() * sizeof(T));          // never-shipped bytes are garbage on a device
        if (host.size()) std::memcpy(static_cast<void*>(v.data()), host.data(), host.size() * sizeof(T));
        up = host.size(); have = true;
    }
    template <class H> void patch(const H& host, std::vector<u32>& dirty) {
        for (u32 i : dirty) v[i] = host[i];
        dirty.clear();
    }
    template <class H> void table(const H& host, bool& full, std::vector<u32>& dirty) {       // engine.cu upload_table
        if (full || !have || up != host.size() || dirty.size() * 8 > host.size()) { fresh(host, 0); dirty.clear(); }
        else patch(host, dirty);
        full = false;
    }
    template <class H> void appendable(const H& host, std::vector<u32>* dirty) {              // engine.cu upload_appendable
        if ((up == 0 && (host.size() > 0 || !have)) || host.size() > v.size()) { fresh(host, std::max(host.size() * 2, size_t(1024))); if (dirty) dirty->clear(); return; }
        const size_t before = up;
        if (host.size() > up) { std::memcpy(static_cast<void*>(v.data() + up), host.data() + up, (host.size() - up) * sizeof(T)); up = host.size(); }
        if (dirty) {
            dirty->erase(std::remove_if(dirty->begin(), dirty->end(), [&](u32 i) { return i >= before; }), dirty->end());
            patch(host, *dirty);
        }
    }
};

struct EmuEngine {
    HostTrie trie{128};
    RetainTreeHost rtree{&trie};
    u32 pool_rows = 24;                  // engine.cu K2_POOL_ROWS (tests lower it to push topics onto the deferred kernel)
    u32 site_bits = 10;
    // optional device image (emu_use_image): the kernels then read copies that only flush() updates
    bool image = false, manual_flush = false;
    ImgBuf<EdgeSlot> i_edges; ImgBuf<DictSlot> i_dict; ImgBuf<Range> i_ranges; ImgBuf<u32> i_values, i_cfilter, i_tree_slots, i_rvals; ImgBuf<u8> i_pool;
    ImgBuf<RKid> i_rkids; ImgBuf<REdge> i_redges;
    u64 up_values_epoch = 0;
    TrieView dev_view{}; RetainView dev_rview{};
    u64 flushes = 0;
    std::vector<u64> last_tasks;         // the last successful retained lookup: tasks queued per round (entry 0 = k_retain_init)
    u64 last_n_desc = 0;                 // ... and descriptors emitted

    bool flush() {                       // engine.cu gm_engine::flush_impl, shipping policy only
        if (!trie.any_dirty() && !rtree.dirty && flushes) return true;
        if (!trie.sync()) return false;
        if (trie.values_epoch != up_values_epoch) { i_values.up = i_ranges.up = 0; up_values_epoch = trie.values_epoch; }
        if (rtree.dirty || !flushes) {
            rtree.prepare_flush();
            if (rtree.full || !i_rkids.have) { i_rkids.fresh(rtree.rkids, rtree.rkids.size() + rtree.rkids.size() / 4 + 1024); i_redges.fresh(rtree.redges, 0); i_rvals.fresh(rtree.rvals, rtree.rvals.size() + 1024); }
            else {
                bool full_edges = false;
                i_rkids.appendable(rtree.rkids, &rtree.dirty_kids);
                i_redges.table(rtree.redges, full_edges, rtree.dirty_edges);
                i_rvals.appendable(rtree.rvals, &rtree.dirty_vals);
            }
            rtree.shipped();
        }
        i_edges.table(trie.edges, trie.full_edges, trie.dirty_edges);
        i_dict.table(trie.dict, trie.full_dict, trie.dirty_dict);
        i_ranges.appendable(trie.ranges, nullptr);
        i_values.appendable(trie.values, nullptr);
        i_pool.appendable(trie.pool, nullptr);
        if (trie.cfilter_dirty || !i_cfilter.have) { i_cfilter.fresh(trie.cfilter, 0); trie.cfilter_dirty = false; }
        if (trie.trees_dirty || !i_tree_slots.have) { i_tree_slots.fresh(trie.tree_slots, 0); trie.trees_dirty = false; }
        trie.root_dirty = false;
        dev_view = host_view();
        dev_view.edges = i_edges.v.data(); dev_view.ranges = i_ranges.v.data(); dev_view.values = i_values.v.data(); dev_view.dict = i_dict.v.data();
        dev_view.pool = i_pool.v.data(); dev_view.cfilter = i_cfilter.v.data(); dev_view.tree_slots = i_tree_slots.v.data();
        dev_rview = host_rview();
        dev_rview.kids = i_rkids.v.data(); dev_rview.edges = i_redges.v.data(); dev_rview.vals = i_rvals.v.data();
        flushes++;
        return true;
    }
    // what a match sees: the live host arrays, or — with the device image — the copies as of the last flush (auto-flush engines
    // flush before every match, GM_FLAG_MANUAL_FLUSH ones only when told to)
    bool prepare(bool retained) {
        if (!image) { if (!trie.sync()) return false; if (retained) { rtree.prepare_flush(); rtree.shipped(); } return true; }
        if (!manual_flush || !flushes) return flush();
        return true;
    }
    TrieView view() { return image ? dev_view : host_view(); }
    RetainView rview() { return image ? dev_rview : host_rview(); }

    TrieView host_view() {               // engine.cu gm_engine::view(), host pointers instead of device pointers
        TrieView v{};
        v.edges = trie.edges.data(); v.ranges = trie.ranges.data(); v.values = trie.values.data(); v.dict = trie.dict.data(); v.pool = trie.pool.data();
        v.cfilter = trie.cfilter.data(); v.cfilter_mask = static_cast<u32>(trie.cfilter.size() - 1);
        v.edge_mask = static_cast<u32>(trie.edges.size() - 1);
        v.win_mask = trie.win_mask(); v.win_shift = trie.win_shift(); v.nwin_mask = trie.nwin_mask();
        v.dict_mask = static_cast<u32>(trie.dict.size() - 1);
        v.root_plus = trie.root_plus; v.root_hash_ref = trie.root_hash_ref; v.root_hash_cnt = trie.root_hash_cnt; v.root_mask = trie.root_mask;
        v.max_depth = trie.max_depth;
        v.tree_slots = trie.tree_slots.data(); v.n_trees = static_cast<u32>(trie.tree_slots.size());
        return v;
    }
    RetainView host_rview() {            // engine.cu gm_engine::rview()
        RetainView v{};
        v.kids = rtree.rkids.data(); v.edges = rtree.redges.data(); v.vals = rtree.rvals.data();
        v.edge_mask = static_cast<u32>(rtree.redges.size() - 1);
        if (!rtree.rnodes.empty()) { v.root_first_kid = rtree.rnodes[0].first_kid; v.root_nk_flags = rtree.rnodes[0].nkids | (rtree.rnodes[0].flags << 28); }
        v.root_plain_kids = rtree.root_plain_kids; v.root_plain_val_hi = rtree.root_plain_val_hi; v.max_depth = rtree.max_depth;
        v.n_kids = static_cast<u32>(rtree.rkids.size());
        return v;
    }
};

}  // namespace

extern "C" {

void* emu_new() { return new EmuEngine(); }
void emu_free(void* h) { delete static_cast<EmuEngine*>(h); }
void emu_set_pool_rows(void* h, uint32_t rows) { static_cast<EmuEngine*>(h)->pool_rows = rows; }
// the kernels read a device IMAGE that only flushes update (manual != 0: only emu_flush, like GM_FLAG_MANUAL_FLUSH)
void emu_use_image(void* h, uint32_t manual) { EmuEngine* e = static_cast<EmuEngine*>(h); e->image = true; e->manual_flush = manual != 0; }
void emu_retain_counters(void* h, uint64_t* out6) { uint64_t o[6]; static_cast<EmuEngine*>(h)->rtree.debug_stats(o); std::memcpy(out6, o, sizeof(o)); }   // {full rebuilds, in-place patches, ...}
int32_t emu_flush(void* h) { return static_cast<EmuEngine*>(h)->flush() ? 0 : -7; }
int32_t emu_compact(void* h) {           // gm_compact: dictionary + value compaction, the retained tree re-labelled
    EmuEngine* e = static_cast<EmuEngine*>(h);
    const std::vector<u32> keep = e->rtree.used_tokens();
    std::vector<u32> remap;
    e->trie.compact(&keep, &remap);
    e->rtree.remap_tokens(remap);
    e->i_ranges.up = e->i_values.up = e->i_pool.up = 0; e->up_values_epoch = e->trie.values_epoch;
    e->i_edges.have = e->i_dict.have = false;
    return 0;
}

int32_t emu_sub_add(void* h, const char* f, uint32_t len, uint32_t value, uint32_t tree) {
    bool ch = false;
    return static_cast<EmuEngine*>(h)->trie.insert(f, len, value, &ch, tree);
}
int32_t emu_sub_remove(void* h, const char* f, uint32_t len, uint32_t value, uint32_t tree) {
    bool ch = false;
    return static_cast<EmuEngine*>(h)->trie.remove(f, len, value, &ch, tree);
}
int32_t emu_retain_set(void* h, const char* t, uint32_t len, uint32_t value) {
    bool had; u32 old;
    return static_cast<EmuEngine*>(h)->rtree.set(t, len, value, &had, &old);
}
int32_t emu_retain_remove(void* h, const char* t, uint32_t len) {
    bool had; u32 old;
    return static_cast<EmuEngine*>(h)->rtree.remove(t, len, &had, &old);
}

// gm_bulk_load / gm_retain_bulk_load: the all-host-threads builds (host_trie.cpp insert_batch_parallel, retain_tree.cpp set_batch_build)
uint64_t emu_bulk_load(void* h, const char* blob, const uint32_t* offs, const uint32_t* vals, uint64_t n) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    e.trie.reserve(n);
    return e.trie.insert_batch(blob, offs, vals, n);
}
uint64_t emu_retain_bulk_load(void* h, const char* blob, const uint32_t* offs, const uint32_t* vals, uint64_t n) {
    return static_cast<EmuEngine*>(h)->rtree.set_batch(blob, offs, vals, n);
}

// Router::matches for a batch through k_tokenize -> k_bucket_scan -> k_bucket_scatter -> k_match_fast -> k_match_slow.
// flags: bit 0 descriptor mode (the descriptors are expanded here from the host mirror, so `out_ids` holds ids either way),
//        bit 1 the bulk-staged tokeniser, bit 2 the instrumented (STATS) instantiations; work[4] = V, E, F, M then.
// Returns 0, or -3 with *needed when cap_ids is too small (the engine's capacity protocol).
//        bit 3 the batch is a SELECTION: row t matches entry sel[t] of the packed batch (n rows, n_entries entries; gm_match_args.d_sel),
//        bit 4 the small-batch-graph form: the kernels are launched for a CAPACITY larger than the batch and read the real
//              batch size / text length from a header in memory (engine.cu small_graph_match).
int32_t emu_match_ex(void* h, const char* blob_in, const uint32_t* offs, uint64_t n_entries, const uint32_t* sel, uint64_t n64, const uint32_t* trees, uint32_t flags,
                     gm_span* out_spans, uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed, int32_t* status, uint64_t* work, uint32_t* deferred) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    const bool desc = flags & 1u, bulk = flags & 2u, stats = flags & 4u, graph_form = flags & 16u;
    if (!(flags & 8u)) sel = nullptr;
    const u32 n_real = static_cast<u32>(n64);
    *needed = 0;
    if (n_real == 0) return 0;
    if (!e.prepare(false)) return -7;
    const TrieView tv = e.view();
    const u32 blob_bytes = offs[n_entries];
    const u32 n = graph_form ? n_real + 37u : n_real;            // launch size (rows beyond the real batch must stay untouched)
    u32 hdr_store[4] = {n_real, blob_bytes, 0u, 0u};
    const u32* hdr = graph_form ? hdr_store : nullptr;
    std::vector<u32> offs_cap;
    if (graph_form) {                                             // the in-block holds capacity + 1 offsets; the tail is never read
        offs_cap.assign(offs, offs + n_entries + 1);
        offs_cap.resize(static_cast<size_t>(n) + 1, 0xDEADBEEFu);
        offs = offs_cap.data();
    }
    // the bulk stage wants a 16-byte aligned blob that may be read up to a 16-byte boundary
    const size_t readable = (static_cast<size_t>(blob_bytes) + 15) & ~size_t(15);
    std::vector<u8> blob_store(readable + 64, 0);
    u8* blob = blob_store.data() + ((16 - (reinterpret_cast<uintptr_t>(blob_store.data()) & 15)) & 15);
    std::memcpy(blob, blob_in, blob_bytes);
    const u32 S = std::max<u32>(1u, tv.max_depth);
    std::vector<u32> tok(S > TOK8 ? static_cast<size_t>(S) * n : 64), meta(n), slow(n);
    std::vector<u32> tok8_store(static_cast<size_t>(n) * TOK8 + 16), sort_store(static_cast<size_t>(n) * 11 + 64);
    u32* tok8 = tok8_store.data() + ((32 - (reinterpret_cast<uintptr_t>(tok8_store.data()) & 31)) & 31) / 4;
    u32* sortb = sort_store.data() + ((32 - (reinterpret_cast<uintptr_t>(sort_store.data()) & 31)) & 31) / 4;
    Ctrl ctrl{};
    const u32 NB = 1u << e.site_bits;
    std::vector<u32> hist_store(2 * static_cast<size_t>(NB) + 16, 0);
    u32* hist = hist_store.data() + ((16 - (reinterpret_cast<uintptr_t>(hist_store.data()) & 15)) & 15) / 4;
    u32* bcursor = hist + NB;
    u32* bkey = sortb; u32* perm = bkey + n; u32* meta_sorted = perm + n;
    u32* tok8_sorted = meta_sorted + n + ((8 - (3 * static_cast<size_t>(n)) % 8) % 8);
    const u32 stack_cap = 32u * (tv.max_depth + 2u) + 64u;
    const int k3_blocks = EMU_SMS * 4;
    std::vector<u64> gstack(static_cast<size_t>(k3_blocks) * 8 * stack_cap);
    const int k2_grid = EMU_SMS * K2_CTAS_PER_SM;
    std::vector<Desc> gpool(static_cast<size_t>(k2_grid) * K2_THREADS * std::max<u32>(e.pool_rows, 1u));
    std::vector<uint2> descs;
    std::vector<u32> ids_tmp;
    void* d_out = out_ids;
    u64 cap = cap_ids;
    if (desc) { descs.resize(cap_ids + 1); d_out = descs.data(); }

    std::vector<int32_t> status_cap;
    int32_t* status_k = status;
    if (graph_form) { status_cap.assign(n, 0x7F7F7F7F); status_k = status_cap.data(); }
    for (u32 i = 0; i < n_real; ++i) status[i] = 0x7F7F7F7F;   // every row must be written by the tokeniser
    emu::launch(dim3((n + TOK_THREADS - 1) / TOK_THREADS), dim3(TOK_THREADS), [&] {
        if (bulk) k_tokenize<true>(blob, blob_bytes, static_cast<u32>(readable), offs, sel, n, hdr, tv, S, tok8, tok.data(), meta.data(), status_k, bkey, hist, e.site_bits, 0u);
        else k_tokenize<false>(blob, blob_bytes, static_cast<u32>(readable), offs, sel, n, hdr, tv, S, tok8, tok.data(), meta.data(), status_k, bkey, hist, e.site_bits, 0u);
    });
    emu::launch(dim3(1), dim3(1024), [&] { k_bucket_scan(hist, bcursor, NB); });
    emu::launch(dim3((n + 255) / 256), dim3(256), [&] { k_bucket_scatter(bkey, bcursor, n, hdr, perm, tok8, meta.data(), tok8_sorted, meta_sorted); });
    if (graph_form) {
        for (u32 i = n_real; i < n; ++i) if (status_cap[i] != 0x7F7F7F7F) return -50;      // a row beyond the real batch was touched
        std::memcpy(status, status_cap.data(), n_real * sizeof(int32_t));
    }
    std::vector<gm_span> spans_cap;
    gm_span* spans_k = out_spans;
    if (graph_form) { spans_cap.assign(n, gm_span{0xABABABABu, 0xABABABABu}); spans_k = spans_cap.data(); }

    MatchParams mp{};
    mp.tv = tv; mp.tok8 = tok8; mp.tok = tok.data(); mp.meta = meta.data(); mp.n = n; mp.n_ptr = hdr; mp.tok_levels = S;
    mp.spans = reinterpret_cast<uint2*>(spans_k); mp.out_ids = static_cast<u32*>(d_out); mp.out_desc = static_cast<uint2*>(d_out); mp.cap_ids = cap;
    mp.status = status_k; mp.trees = trees;
    mp.cursor = &ctrl.cursor; mp.slow_list = slow.data(); mp.slow_count = &ctrl.slow_count; mp.tile_counter = &ctrl.tile_counter; mp.stats = ctrl.stats;
    mp.perm = perm; mp.tok8_sorted = tok8_sorted; mp.meta_sorted = meta_sorted;
    mp.flags = MP_SORTED_ROWS; mp.tile_chunk = 1;
    emu::launch(dim3(k2_grid), dim3(K2_THREADS), [&] {
        if (stats) { if (desc) k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, true, true>(mp, gpool.data(), e.pool_rows); else k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, true, false>(mp, gpool.data(), e.pool_rows); }
        else { if (desc) k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, false, true>(mp, gpool.data(), e.pool_rows); else k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, false, false>(mp, gpool.data(), e.pool_rows); }
    });
    emu::launch(dim3(k3_blocks), dim3(256), [&] {
        if (stats) { if (desc) k_match_slow<true, true>(mp, gstack.data(), stack_cap); else k_match_slow<true, false>(mp, gstack.data(), stack_cap); }
        else { if (desc) k_match_slow<false, true>(mp, gstack.data(), stack_cap); else k_match_slow<false, false>(mp, gstack.data(), stack_cap); }
    });
    if (graph_form) {
        for (u32 i = n_real; i < n; ++i) if (spans_cap[i].off != 0xABABABABu) return -51;
        std::memcpy(out_spans, spans_cap.data(), n_real * sizeof(gm_span));
    }
    if (deferred) *deferred = ctrl.slow_count;
    if (work) for (int k = 0; k < 4; ++k) work[k] = ctrl.stats[k];
    *needed = ctrl.cursor;
    if (ctrl.cursor > cap_ids) return -3;
    if (!desc) return 0;
    // descriptor mode: expand (ref, cnt) into ids out of the host mirror, per topic, so that the caller compares id lists
    u64 w = 0;
    for (u32 t = 0; t < n_real; ++t) {
        const u32 off = out_spans[t].off, cnt = out_spans[t].cnt;
        const u64 begin = w;
        for (u32 k = 0; k < cnt; ++k) {
            const uint2 d = descs[off + k];
            if (d.y == 1) ids_tmp.push_back(d.x);
            else {
                u64 o = d.x, c = d.y;
                if (d.y == CNT_BIG) { o = e.trie.ranges[d.x].off; c = e.trie.ranges[d.x].cnt; }
                for (u64 j = 0; j < c; ++j) ids_tmp.push_back(e.trie.values[o + j]);
            }
        }
        w = ids_tmp.size();
        out_spans[t] = gm_span{static_cast<u32>(begin), static_cast<u32>(w - begin)};
    }
    *needed = w;                      // (in descriptor mode the capacity the caller must offer is the expanded size)
    if (w > cap_ids) return -3;
    std::memcpy(out_ids, ids_tmp.data(), w * sizeof(u32));
    return 0;
}

int32_t emu_match(void* h, const char* blob_in, const uint32_t* offs, uint64_t n64, const uint32_t* trees, uint32_t flags, gm_span* out_spans, uint32_t* out_ids,
                  uint64_t cap_ids, uint64_t* needed, int32_t* status, uint64_t* work, uint32_t* deferred) {
    return emu_match_ex(h, blob_in, offs, n64, nullptr, n64, trees, flags & ~8u, out_spans, out_ids, cap_ids, needed, status, work, deferred);
}

// gm_partition_batch_device: k_partition.  counts[n_shards + 1] (the last entry = rows appended to sel)
int32_t emu_partition(const char* blob, const uint32_t* offs, uint64_t n, uint32_t n_shards, uint32_t rank, uint32_t* sel, uint32_t* shard_out, uint32_t* counts) {
    std::memset(counts, 0, (static_cast<size_t>(n_shards) + 1) * sizeof(u32));
    if (n == 0) return 0;
    const u32 blob_bytes = offs[n];
    emu::launch(dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), [&] {
        k_partition(reinterpret_cast<const u8*>(blob), blob_bytes, offs, static_cast<u32>(n), n_shards, rank, sel, shard_out, counts);
    });
    return 0;
}

// ---- the fused gather over "peer memory": every rank's block lives in host memory of this one process ---------------------------
struct GatherWorld {
    u32 world = 0; u64 slab_topics = 0, slab_ids = 0;
    static constexpr size_t off_ids = 256;
    size_t off_spans = 0, off_index = 0, off_counts = 0, off_flags = 0, bytes = 0;
    std::vector<std::vector<char>> store;
    std::vector<char*> block;
    std::vector<u32> epoch;
    std::vector<unsigned long long> cursor;      // the match cursor of every rank's last step (k_gather_push / k_gather_finish read it)
};
void* emu_gather_new(uint32_t world, uint64_t slab_topics, uint64_t slab_ids) {       // engine.cu gm_gather_create's layout
    GatherWorld* g = new GatherWorld();
    slab_topics = (slab_topics + 3) & ~uint64_t(3); slab_ids = (slab_ids + 3) & ~uint64_t(3);
    g->world = world; g->slab_topics = slab_topics; g->slab_ids = slab_ids;
    const size_t a = 256;
    g->off_spans = (GatherWorld::off_ids + static_cast<size_t>(world) * slab_ids * 4 + a - 1) / a * a;
    g->off_index = g->off_spans + static_cast<size_t>(world) * slab_topics * 8;
    g->off_counts = (g->off_index + static_cast<size_t>(world) * slab_topics * 4 + a - 1) / a * a;
    g->off_flags = g->off_counts + static_cast<size_t>(world) * 16;
    g->bytes = g->off_flags + 256;
    g->store.resize(world); g->block.resize(world); g->epoch.assign(world, 0); g->cursor.assign(world, 0);
    for (u32 w = 0; w < world; ++w) {
        g->store[w].assign(g->bytes + 256, static_cast<char>(0xEE));        // (stale bytes must never be read as results)
        g->block[w] = g->store[w].data() + ((256 - (reinterpret_cast<uintptr_t>(g->store[w].data()) & 255)) & 255);
        std::memset(g->block[w] + g->off_counts, 0, g->bytes - g->off_counts);
    }
    return g;
}
void emu_gather_free(void* p) { delete static_cast<GatherWorld*>(p); }
uint64_t emu_gather_slab_ids(void* p) { return static_cast<GatherWorld*>(p)->slab_ids; }
uint64_t emu_gather_slab_topics(void* p) { return static_cast<GatherWorld*>(p)->slab_topics; }

// gm_match_gather_device of ONE rank: its rows (sel / n) through the GATHER instantiations of the match kernels, then — push form —
// k_gather_push copies the rank's slab into every peer's block.  direct != 0: the publish phase stores into every block itself.
int32_t emu_match_gather(void* gw, uint32_t rank, void* h, const char* blob_in, const uint32_t* offs, uint64_t n_entries, const uint32_t* sel, uint64_t n64,
                         uint32_t direct, int32_t* status) {
    GatherWorld& G = *static_cast<GatherWorld*>(gw);
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    const u32 n = static_cast<u32>(n64);
    if (n > G.slab_topics) return -3;
    G.cursor[rank] = 0;
    if (n) {
        if (!e.prepare(false)) return -7;
        const TrieView tv = e.view();
        const u32 blob_bytes = offs[n_entries];
        const size_t readable = (static_cast<size_t>(blob_bytes) + 15) & ~size_t(15);
        std::vector<u8> blob_store(readable + 64, 0);
        u8* blob = blob_store.data() + ((16 - (reinterpret_cast<uintptr_t>(blob_store.data()) & 15)) & 15);
        std::memcpy(blob, blob_in, blob_bytes);
        const u32 S = std::max<u32>(1u, tv.max_depth);
        std::vector<u32> tok(S > TOK8 ? static_cast<size_t>(S) * n : 64), meta(n), slow(n);
        std::vector<u32> tok8_store(static_cast<size_t>(n) * TOK8 + 16), sort_store(static_cast<size_t>(n) * 11 + 64);
        u32* tok8 = tok8_store.data() + ((32 - (reinterpret_cast<uintptr_t>(tok8_store.data()) & 31)) & 31) / 4;
        u32* sortb = sort_store.data() + ((32 - (reinterpret_cast<uintptr_t>(sort_store.data()) & 31)) & 31) / 4;
        Ctrl ctrl{};
        const u32 NB = 1u << e.site_bits;
        std::vector<u32> hist_store(2 * static_cast<size_t>(NB) + 16, 0);
        u32* hist = hist_store.data() + ((16 - (reinterpret_cast<uintptr_t>(hist_store.data()) & 15)) & 15) / 4;
        u32* bcursor = hist + NB;
        u32* bkey = sortb; u32* perm = bkey + n; u32* meta_sorted = perm + n;
        u32* tok8_sorted = meta_sorted + n + ((8 - (3 * static_cast<size_t>(n)) % 8) % 8);
        const u32 stack_cap = 32u * (tv.max_depth + 2u) + 64u;
        const int k3_blocks = EMU_SMS * 4, k2_grid = EMU_SMS * K2_CTAS_PER_SM;
        std::vector<u64> gstack(static_cast<size_t>(k3_blocks) * 8 * stack_cap);
        std::vector<Desc> gpool(static_cast<size_t>(k2_grid) * K2_THREADS * std::max<u32>(e.pool_rows, 1u));
        emu::launch(dim3((n + TOK_THREADS - 1) / TOK_THREADS), dim3(TOK_THREADS), [&] {
            k_tokenize<false>(blob, blob_bytes, static_cast<u32>(readable), offs, sel, n, nullptr, tv, S, tok8, tok.data(), meta.data(), status, bkey, hist, e.site_bits, 0u);
        });
        emu::launch(dim3(1), dim3(1024), [&] { k_bucket_scan(hist, bcursor, NB); });
        emu::launch(dim3((n + 255) / 256), dim3(256), [&] { k_bucket_scatter(bkey, bcursor, n, nullptr, perm, tok8, meta.data(), tok8_sorted, meta_sorted); });
        MatchParams mp{};
        mp.tv = tv; mp.tok8 = tok8; mp.tok = tok.data(); mp.meta = meta.data(); mp.n = n; mp.tok_levels = S;
        mp.cap_ids = G.slab_ids; mp.status = status;
        mp.cursor = &ctrl.cursor; mp.slow_list = slow.data(); mp.slow_count = &ctrl.slow_count; mp.tile_counter = &ctrl.tile_counter; mp.stats = ctrl.stats;
        mp.perm = perm; mp.tok8_sorted = tok8_sorted; mp.meta_sorted = meta_sorted;
        mp.flags = MP_SORTED_ROWS; mp.tile_chunk = 1;
        mp.g_base_topics = static_cast<u32>(rank * G.slab_topics); mp.g_base_ids = rank * G.slab_ids; mp.g_sel = sel;     // engine.cu enqueue_match, gather_mode
        if (direct) {
            mp.g_world = G.world;
            for (u32 w = 0; w < G.world; ++w) {
                mp.g_ids[w] = reinterpret_cast<u32*>(G.block[w] + GatherWorld::off_ids); mp.g_spans[w] = reinterpret_cast<uint2*>(G.block[w] + G.off_spans);
                mp.g_index[w] = reinterpret_cast<u32*>(G.block[w] + G.off_index);
            }
        } else {
            mp.g_world = 1;
            mp.g_ids[0] = reinterpret_cast<u32*>(G.block[rank] + GatherWorld::off_ids); mp.g_spans[0] = reinterpret_cast<uint2*>(G.block[rank] + G.off_spans);
            mp.g_index[0] = reinterpret_cast<u32*>(G.block[rank] + G.off_index);
        }
        emu::launch(dim3(k2_grid), dim3(K2_THREADS), [&] { k_match_fast<K2_FAST_L, K2_THREADS, K2_CTAS_PER_SM, false, false, true>(mp, gpool.data(), e.pool_rows); });
        emu::launch(dim3(k3_blocks), dim3(256), [&] { k_match_slow<false, false, true>(mp, gstack.data(), stack_cap); });
        G.cursor[rank] = ctrl.cursor;
        if (ctrl.cursor > G.slab_ids) return -3;
    }
    if (!direct && G.world > 1)
        emu::launch(dim3(EMU_SMS * 4), dim3(256), [&] {
            k_gather_push(G.block.data(), rank, G.world, GatherWorld::off_ids, G.off_spans, G.off_index, rank * G.slab_topics, rank * G.slab_ids, n, &G.cursor[rank]);
        });
    return 0;
}

// the end-of-step kernel of one rank (counts + flag to every block, bounded wait for the others' flags); returns the rank's error word
int32_t emu_gather_finish(void* gw, uint32_t rank, uint64_t n, uint32_t new_epoch) {
    GatherWorld& G = *static_cast<GatherWorld*>(gw);
    if (new_epoch) G.epoch[rank]++;
    std::vector<unsigned long long*> counts(G.world);
    std::vector<u32*> flags(G.world);
    for (u32 w = 0; w < G.world; ++w) { counts[w] = reinterpret_cast<unsigned long long*>(G.block[w] + G.off_counts); flags[w] = reinterpret_cast<u32*>(G.block[w] + G.off_flags); }
    u32* my_flags = reinterpret_cast<u32*>(G.block[rank] + G.off_flags);
    my_flags[32] = 0;                                                                 // the error word
    emu::launch(dim3(1), dim3(32), [&] { k_gather_finish(counts.data(), flags.data(), my_flags, rank, G.world, n, &G.cursor[rank], G.epoch[rank], my_flags + 32); });
    return static_cast<int32_t>(my_flags[32]);
}

// one rank's view of the gathered arrays (gm_gather_get + the copies Engine.gather_result makes)
void emu_gather_read(void* gw, uint32_t rank, uint64_t* counts, uint32_t* index, gm_span* spans, uint32_t* ids) {
    GatherWorld& G = *static_cast<GatherWorld*>(gw);
    const char* b = G.block[rank];
    std::memcpy(counts, b + G.off_counts, static_cast<size_t>(G.world) * 16);
    std::memcpy(index, b + G.off_index, static_cast<size_t>(G.world) * G.slab_topics * 4);
    std::memcpy(spans, b + G.off_spans, static_cast<size_t>(G.world) * G.slab_topics * 8);
    std::memcpy(ids, b + GatherWorld::off_ids, static_cast<size_t>(G.world) * G.slab_ids * 4);
}

// RetainStorage::get for a batch of filters through k_tokenize -> k_retain_init -> k_retain_round x (depth + 1) -> k_retain_scan -> k_retain_expand
int32_t emu_retain_match(void* h, const char* blob_in, const uint32_t* offs, uint64_t n64, uint32_t stats_on, uint32_t cap_items, uint32_t cap_desc, gm_span* out_spans,
                         uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed, int32_t* status, uint64_t* work) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    const u32 nq = static_cast<u32>(n64);
    *needed = 0;
    if (nq == 0) return 0;
    if (!e.prepare(true)) return -7;
    const TrieView tv = e.view();
    const RetainView rv = e.rview();
    const u32 depth = rv.max_depth, S = depth + 2;
    const u32 blob_bytes = offs[nq];
    std::vector<u8> blob_store(static_cast<size_t>(blob_bytes) + 64, 0);
    u8* blob = blob_store.data() + ((16 - (reinterpret_cast<uintptr_t>(blob_store.data()) & 15)) & 15);
    std::memcpy(blob, blob_in, blob_bytes);
    std::vector<u32> tok(S > TOK8 ? static_cast<size_t>(S) * nq : 64), meta(nq);
    std::vector<u32> tok8_store(static_cast<size_t>(nq) * TOK8 + 16);
    u32* tok8 = tok8_store.data() + ((32 - (reinterpret_cast<uintptr_t>(tok8_store.data()) & 31)) & 31) / 4;
    struct RCtl { unsigned long long grand; unsigned long long stats[2]; u32 err; u32 pad; u32 n_desc[RQ]; };
    RCtl ctl{};
    std::vector<u32> counts(static_cast<size_t>(depth + 3) * RQ + (depth + 3), 0);
    std::vector<u32> rq(static_cast<size_t>(nq) * 3, 0);
    u32* qtotal = rq.data(); u32* qbase = qtotal + nq; u32* qcur = qbase + nq;
    const u32 slice_items = std::max<u32>(1u, cap_items / RQ), slice_desc = std::max<u32>(1u, cap_desc / RQ);
    std::vector<RTask> front[2] = {std::vector<RTask>(static_cast<size_t>(slice_items) * RQ), std::vector<RTask>(static_cast<size_t>(slice_items) * RQ)};
    std::vector<RDesc> rdescs(static_cast<size_t>(slice_desc) * RQ);
    for (u32 i = 0; i < nq; ++i) status[i] = 0x7F7F7F7F;
    emu::launch(dim3((nq + TOK_THREADS - 1) / TOK_THREADS), dim3(TOK_THREADS), [&] {
        k_tokenize<false>(blob, blob_bytes, blob_bytes, offs, nullptr, nq, nullptr, tv, S, tok8, tok.data(), meta.data(), status, nullptr, nullptr, 0u, 0u);
    });
    RetainParams rp{};
    rp.v = rv; rp.qtok8 = tok8; rp.qtok = tok.data(); rp.qmeta = meta.data(); rp.nq = nq; rp.tok_levels = S;
    rp.descs = rdescs.data(); rp.n_desc = ctl.n_desc; rp.cap_items = slice_items; rp.cap_desc = slice_desc;
    rp.qtotal = qtotal; rp.err = &ctl.err; rp.stats = ctl.stats;
    emu::launch(dim3((nq + 255) / 256), dim3(256), [&] { if (stats_on) k_retain_init<true>(rp, front[0].data(), &counts[0]); else k_retain_init<false>(rp, front[0].data(), &counts[0]); });
    const int rgrid = EMU_SMS * GM_RETAIN_CTAS;
    for (u32 lvl = 0; lvl <= depth; ++lvl)
        emu::launch(dim3(rgrid), dim3(256), [&] {
            u32* claim = &counts[static_cast<size_t>(depth + 3) * RQ + lvl];
            if (stats_on) k_retain_round<true>(rp, front[lvl & 1].data(), &counts[static_cast<size_t>(lvl) * RQ], front[(lvl + 1) & 1].data(), &counts[static_cast<size_t>(lvl + 1) * RQ], claim);
            else k_retain_round<false>(rp, front[lvl & 1].data(), &counts[static_cast<size_t>(lvl) * RQ], front[(lvl + 1) & 1].data(), &counts[static_cast<size_t>(lvl + 1) * RQ], claim);
        });
    emu::launch(dim3(1), dim3(1024), [&] { k_retain_scan(qtotal, nq, qbase, reinterpret_cast<uint2*>(out_spans), &ctl.grand); });
    emu::launch(dim3(EMU_SMS * 8), dim3(256), [&] { k_retain_expand(rdescs.data(), ctl.n_desc, slice_desc, rv.vals, qbase, qcur, out_ids, cap_ids); });
    if (work) { work[0] = ctl.stats[0]; work[1] = ctl.stats[1]; }
    if (ctl.err) return -100 - static_cast<int32_t>(ctl.err);      // scratch overflow: bit 0 tasks, bit 1 descriptors (the engine grows and retries)
    e.last_tasks.assign(depth + 2, 0);                             // the totals of engine.cu's `retain stats` line
    for (u32 l = 0; l <= depth + 1; ++l) for (u32 k = 0; k < RQ; ++k) e.last_tasks[l] += counts[static_cast<size_t>(l) * RQ + k];
    e.last_n_desc = 0;
    for (u32 k = 0; k < RQ; ++k) e.last_n_desc += ctl.n_desc[k];
    *needed = ctl.grand;
    return ctl.grand > cap_ids ? -3 : 0;
}

// tasks queued per round by the last successful emu_retain_match (entry 0 = k_retain_init, entry l + 1 = round l) into
// out[0 .. cap); returns the number of rounds + 1 (max_depth + 2); *n_desc = the descriptors it emitted
uint32_t emu_retain_last_tasks(void* h, uint64_t* out, uint32_t cap, uint64_t* n_desc) {
    const EmuEngine& e = *static_cast<EmuEngine*>(h);
    for (size_t l = 0; l < e.last_tasks.size() && l < cap; ++l) out[l] = e.last_tasks[l];
    if (n_desc) *n_desc = e.last_n_desc;
    return static_cast<uint32_t>(e.last_tasks.size());
}
// the host image of the retained tree (gm_debug_table 7 = rnodes, 8 = rkids: 8 words per entry)
int32_t emu_retain_table(void* h, uint32_t which, const void** ptr, uint64_t* count) {
    RetainTreeHost& t = static_cast<EmuEngine*>(h)->rtree;
    t.prepare_flush();
    if (which == 7) { *ptr = t.rnodes.data(); *count = t.rnodes.size(); }
    else if (which == 8) { *ptr = t.rkids.data(); *count = t.rkids.size(); }
    else return -1;
    return 0;
}

// gm_relations_expand_device over host arrays (k_relations)
int32_t emu_relations(const gm_span* spans, const uint32_t* ids, uint64_t n, const uint32_t* pubs, const gm_rel* rels, uint64_t n_rels, gm_span* out_spans,
                      gm_sub_relation* out_rels, uint64_t cap_rels, uint32_t* out_sub_ids, uint64_t cap_sub_ids, uint64_t* needed3, int32_t* status) {
    needed3[0] = needed3[1] = needed3[2] = 0;
    if (n == 0) return 0;
    RelParams rp{};
    rp.spans = reinterpret_cast<const uint2*>(spans); rp.ids = ids; rp.n = static_cast<u32>(n); rp.pubs = pubs; rp.rels = rels; rp.n_rels = static_cast<u32>(n_rels);
    rp.out_spans = reinterpret_cast<uint2*>(out_spans); rp.out_rels = out_rels; rp.cap_rels = cap_rels; rp.out_sub_ids = out_sub_ids; rp.cap_sub_ids = cap_sub_ids;
    rp.needed = reinterpret_cast<unsigned long long*>(needed3); rp.status = status;
    const unsigned grid = static_cast<unsigned>(std::min<u64>((n + 7) / 8, static_cast<u64>(EMU_SMS) * 8));
    emu::launch(dim3(grid), dim3(256), [&] { k_relations(rp); });
    return 0;
}

}  // extern "C"
