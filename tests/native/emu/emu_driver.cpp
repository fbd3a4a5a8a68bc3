// TEST INFRASTRUCTURE: the match and retained-lookup pipelines over HOST memory.  The launch sequences, scratch plan, views
// and shipping decisions are engine.cu's own (rmqtt_b200/csrc/pipeline.cuh); the REAL kernel sources (kernels.cuh,
// retain_kernels.cuh, relations.cuh compiled with -DGM_CPU_EMU) run on the CPU emulation in cuda_runtime.h.  What stays here
// is what the engine does around a launch (staging, the device image a flush keeps) and the test-only checks.  Exposed as a
// small C interface for tests/test_emu_kernels.py, which compares the results with the oracle.  Build (the test does it):
//   g++ -O1 -g -std=c++17 -DGM_CPU_EMU -Itests/native/emu -Irmqtt_b200/csrc -shared -fPIC tests/native/emu/emu_driver.cpp \
//       rmqtt_b200/csrc/host_trie.cpp rmqtt_b200/csrc/retain_tree.cpp -o <out>.so     (+ -fsanitize=address,undefined for the ASan run)
#include <cuda_runtime.h>      // the emulation (this directory is first on the include path)

#include <cstring>
#include <memory>
#ifdef EMU_ASAN
#include <sanitizer/asan_interface.h>
#endif
#include <new>
#include <vector>

#include "comm.cuh"
#include "pipeline.cuh"
#include "relations.cuh"

using namespace gm;

namespace {

constexpr u32 EMU_SMS = 2;               // the emulated part has two SMs: several CTAs per kernel, dynamic tile hand-out exercised

// Host memory standing in for cudaMalloc'd scratch, 256-byte aligned.  A fresh block holds POISON, not zeros:
// a device allocation holds garbage, and the engine clears only what pipeline.cuh's match_resets names (retained lookups:
// their control block and queue counters), so a read of scratch the call never wrote shows up as a wrong result.  GUARD bytes follow every block in the same allocation.  In the
// plain build they hold POISON and intact() after the call catches a write past the block's end.  In the ASan build they
// are also marked unaddressable, so ASan still reports any read or write past the block's end, as it would for an
// allocation of exactly the block's size.
constexpr u8 POISON = 0xA5;
constexpr size_t GUARD = 256;
#ifdef EMU_ASAN
inline void guard_off(const void* p, size_t n) { ASAN_UNPOISON_MEMORY_REGION(p, n); }
inline void guard_on(const void* p, size_t n) { ASAN_POISON_MEMORY_REGION(p, n); }
#else
inline void guard_off(const void*, size_t) {}
inline void guard_on(const void*, size_t) {}
#endif
struct Block {
    u8* p = nullptr;
    size_t cap = 0;
    Block() = default;
    Block(const Block&) = delete;
    Block& operator=(const Block&) = delete;
    ~Block() { release(); }
    void release() {
        if (p) { guard_off(p + cap, GUARD); ::operator delete(p, std::align_val_t(256)); }
        p = nullptr;
    }
    // exact: a block of exactly `bytes`; else the engine's DevBuf::ensure: grow (a fresh block) only when too small, keep the contents otherwise
    template <class T> T* get(size_t bytes, bool exact = true, u8 fill = POISON) {
        if (!p || (exact ? bytes != cap : bytes > cap)) {
            const size_t ncap = exact || !p ? bytes : std::max(bytes, cap + cap / 2);
            release();
            cap = ncap;
            p = static_cast<u8*>(::operator new(cap + GUARD, std::align_val_t(256)));
            std::memset(p, fill, cap);
            std::memset(p + cap, POISON, GUARD);
            guard_on(p + cap, GUARD);
        }
        return reinterpret_cast<T*>(p);
    }
    bool intact() const {
        if (!p) return true;
        guard_off(p + cap, GUARD);
        bool ok = true;
        for (size_t i = 0; i < GUARD; ++i) ok &= p[cap + i] == POISON;
        guard_on(p + cap, GUARD);
        return ok;
    }
};
// the retained lookup's scratch: poisoned as well (engine.cu clears its control block and queue counters, as the driver does)
struct Arena {
    std::vector<std::unique_ptr<Block>> blocks;
    template <class T> T* get(size_t bytes) { blocks.emplace_back(new Block()); return blocks.back()->get<T>(bytes); }
    bool intact() const { for (const auto& b : blocks) if (!b->intact()) return false; return true; }
};

// the scratch of one match context (engine.cu MatchCtx): fresh and exactly sized for every call, or kept across calls
struct MatchBufs {
    Block tok, tok8, meta, slow, sort, hist, ctrl, gstack, gpool;
    MatchScratch get(const MatchPlan& p, bool exact) {
        MatchScratch m{};
        m.tok = tok.get<u32>(p.tok, exact); m.tok8 = tok8.get<u32>(p.tok8, exact); m.meta = meta.get<u32>(p.meta, exact); m.slow = slow.get<u32>(p.slow, exact);
        m.sort = sort.get<u32>(p.sort, exact); m.hist = hist.get<u32>(p.hist, exact); m.ctrl = ctrl.get<Ctrl>(p.ctrl, exact); m.gstack = gstack.get<u64>(p.gstack, exact);
        m.gpool = gpool.get<Desc>(p.gpool, exact);
        return m;
    }
    bool intact() const {
        for (const Block* b : {&tok, &tok8, &meta, &slow, &sort, &hist, &ctrl, &gstack, &gpool}) if (!b->intact()) return false;
        return true;
    }
};

// a batch's text, 16-byte aligned and readable up to the next 16-byte boundary (what the bulk tokeniser may read)
struct Text {
    std::vector<u8> store;
    u8* p;
    u32 bytes, readable;
    Text(const char* src, u32 n) : store((static_cast<size_t>(n) + 15) / 16 * 16 + 64, 0), bytes(n), readable((n + 15u) & ~15u) {
        p = store.data() + ((16 - (reinterpret_cast<uintptr_t>(store.data()) & 15)) & 15);
        std::memcpy(p, src, n);
    }
};

// A "device copy" of one table, maintained ONLY by what gm_engine::flush_impl would ship (pipeline.cuh ship_table_whole /
// ship_appendable_fresh): whole arrays, appended tails, and the slots the host mirror listed as dirty.  A slot the mirror
// changed without listing it stays stale here — and shows up as a wrong match.
template <class T> struct ImgBuf {
    std::vector<T> v;                    // v.size() * sizeof(T) plays the role of DevBuf::cap
    size_t up = 0;                       // shipped up to here (appendable arrays) / shipped size (tables)
    bool have = false;
    template <class H> void fresh(const H& host, size_t min_bytes, size_t slack_bytes = 0) {
        v.assign((fresh_bytes(host.size() * sizeof(T), min_bytes, slack_bytes) + sizeof(T) - 1) / sizeof(T), T{});
        std::memset(static_cast<void*>(v.data()), 0xCD, v.size() * sizeof(T));          // never-shipped bytes are garbage on a device
        if (host.size()) std::memcpy(static_cast<void*>(v.data()), host.data(), host.size() * sizeof(T));
        up = host.size(); have = true;
    }
    template <class H> void patch(const H& host, std::vector<u32>& dirty) {
        for (u32 i : dirty) v[i] = host[i];
        dirty.clear();
    }
    template <class H> void table(const H& host, bool& full, std::vector<u32>& dirty) {       // engine.cu upload_table
        if (ship_table_whole(full, up, host.size(), dirty.size())) { fresh(host, 0); dirty.clear(); }
        else patch(host, dirty);
        full = false;
    }
    template <class H> void appendable(const H& host, std::vector<u32>* dirty) {              // engine.cu upload_appendable
        const size_t bytes = host.size() * sizeof(T);
        if (ship_appendable_fresh(up, bytes, have, v.size() * sizeof(T))) { fresh(host, appendable_room(bytes)); if (dirty) dirty->clear(); return; }
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
    u32 pool_rows = K2_POOL_ROWS;        // (tests lower it to push topics onto the deferred kernel)
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
            if (rtree.full || !i_rkids.have) { i_rkids.fresh(rtree.rkids, 0, retained_kids_slack(rtree.rkids.size())); i_redges.fresh(rtree.redges, 0); i_rvals.fresh(rtree.rvals, 0, RETAINED_VALS_SLACK); }
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
        dev_view = trie_view(trie, i_edges.v.data(), i_ranges.v.data(), i_values.v.data(), i_dict.v.data(), i_pool.v.data(), i_cfilter.v.data(), i_tree_slots.v.data());
        dev_rview = retain_view(rtree, i_rkids.v.data(), i_redges.v.data(), i_rvals.v.data());
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
    TrieView view() {
        if (image) return dev_view;
        return trie_view(trie, trie.edges.data(), trie.ranges.data(), trie.values.data(), trie.dict.data(), trie.pool.data(), trie.cfilter.data(), trie.tree_slots.data());
    }
    RetainView rview() { return image ? dev_rview : retain_view(rtree, rtree.rkids.data(), rtree.redges.data(), rtree.rvals.data()); }

    // scheduling knobs (gm_debug_knob) and the launch capacity of the small-graph form (0: the batch size + 37)
    u32 tile_chunk = 1, diag_flags = 0, graph_cap = 0;
    int k2_ctas = 0;
    // keep_scratch: one scratch across calls, as a match context keeps it (grown only when too small); else a fresh one per call
    bool keep_scratch = false;
    MatchBufs kept;
    bool overrun = false;                // a call wrote past the end of a scratch block (its guard bytes changed)

    // one match through engine.cu's launch sequence, its scratch allocated by the plan and cleared as the engine clears it;
    // returns the control block
    Ctrl match(const MatchIO& io, bool bulk, bool keep_cursor = false) {
        const TrieView tv = view();
        MatchKnobs kn;
        kn.tok_bulk = bulk; kn.site_bits = site_bits; kn.pool_rows = pool_rows;
        kn.tile_chunk = tile_chunk; kn.k2_ctas = k2_ctas; kn.diag_flags = diag_flags;
        const MatchPlan p = plan_match(static_cast<u32>(io.n), tv.max_depth, kn, EMU_SMS, io.hdr != nullptr);
        MatchBufs fresh;
        MatchBufs& b = keep_scratch ? kept : fresh;
        const MatchScratch m = b.get(p, !keep_scratch);
        for (const ByteRange& r : match_resets(p, m, keep_cursor).r) std::memset(r.p, 0, r.bytes);
        launch_match(p, m, io, kn, tv, nullptr);
        if (!b.intact()) overrun = true;
        return *m.ctrl;
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
    e->i_edges.up = e->i_dict.up = 0;
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
//        bit 5 (with bit 0) raw descriptors: out_ids receives cap_ids descriptors (ref, cnt) as the kernels wrote them, unexpanded.
// -60: a kernel wrote past the end of a scratch block.
int32_t emu_match_ex(void* h, const char* blob_in, const uint32_t* offs, uint64_t n_entries, const uint32_t* sel, uint64_t n64, const uint32_t* trees, uint32_t flags,
                     gm_span* out_spans, uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed, int32_t* status, uint64_t* work, uint32_t* deferred) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    const bool desc = flags & 1u, graph_form = flags & 16u, raw_desc = desc && (flags & 32u);
    if (!(flags & 8u)) sel = nullptr;
    const u32 n_real = static_cast<u32>(n64);
    *needed = 0;
    if (n_real == 0) return 0;
    if (!e.prepare(false)) return -7;
    const Text text(blob_in, offs[n_entries]);
    if (graph_form && e.graph_cap && e.graph_cap < n_real) return -2;
    const u32 n = graph_form ? (e.graph_cap ? e.graph_cap : n_real + 37u) : n_real;   // launch size (rows beyond the real batch must stay untouched)
    const u32 hdr[4] = {n_real, text.bytes, 0u, 0u};
    std::vector<u32> offs_cap;
    if (graph_form) {                                             // the in-block holds capacity + 1 offsets; the tail is never read
        offs_cap.assign(offs, offs + n_entries + 1);
        offs_cap.resize(static_cast<size_t>(n) + 1, 0xDEADBEEFu);
        offs = offs_cap.data();
    }
    std::vector<uint2> descs;
    if (desc && !raw_desc) descs.resize(cap_ids + 1);
    std::vector<int32_t> status_cap;
    std::vector<gm_span> spans_cap;
    for (u32 i = 0; i < n_real; ++i) status[i] = 0x7F7F7F7F;   // every row must be written by the tokeniser
    if (graph_form) { status_cap.assign(n, 0x7F7F7F7F); spans_cap.assign(n, gm_span{0xABABABABu, 0xABABABABu}); }

    MatchIO io;
    io.blob = text.p; io.blob_bytes = text.bytes; io.readable_bytes = text.readable; io.offs = offs; io.sel = sel; io.n = n; io.trees = trees;
    io.hdr = graph_form ? hdr : nullptr;
    io.spans = graph_form ? spans_cap.data() : out_spans; io.status = graph_form ? status_cap.data() : status;
    io.out = desc && !raw_desc ? static_cast<void*>(descs.data()) : out_ids; io.cap = cap_ids;
    io.stats = flags & 4u; io.desc = desc;
    e.overrun = false;
    const Ctrl ctrl = e.match(io, flags & 2u);
    if (e.overrun) return -60;
    if (graph_form) {
        for (u32 i = n_real; i < n; ++i) if (status_cap[i] != 0x7F7F7F7F) return -50;      // a row beyond the real batch was touched
        for (u32 i = n_real; i < n; ++i) if (spans_cap[i].off != 0xABABABABu) return -51;
        std::memcpy(status, status_cap.data(), n_real * sizeof(int32_t));
        std::memcpy(out_spans, spans_cap.data(), n_real * sizeof(gm_span));
    }
    if (deferred) *deferred = ctrl.slow_count;
    if (work) for (int k = 0; k < 4; ++k) work[k] = ctrl.stats[k];
    *needed = ctrl.cursor;
    if (ctrl.cursor > cap_ids) return -3;
    if (!desc || raw_desc) return 0;
    // descriptor mode: expand (ref, cnt) into ids out of the host mirror, per topic, so that the caller compares id lists
    std::vector<u32> ids_tmp;
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

// The pipelined host call (engine.cu match_host_impl): chunks of `chunk` rows, one after the other on ONE kept scratch; the
// first chunk clears the whole control block, every later one all of it but the bump cursor over out_ids (keep_cursor).
// flags: bit 1 the bulk-staged tokeniser.  Returns 0, -3 (*needed: ids needed) or -60 as emu_match_ex.
int32_t emu_match_chunked(void* h, const char* blob_in, const uint32_t* offs, uint64_t n64, uint32_t flags, uint64_t chunk, gm_span* out_spans, uint32_t* out_ids,
                          uint64_t cap_ids, uint64_t* needed, int32_t* status) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    *needed = 0;
    if (n64 == 0) return 0;
    if (chunk == 0) return -2;
    if (!e.prepare(false)) return -7;
    const Text text(blob_in, offs[n64]);
    for (u64 i = 0; i < n64; ++i) status[i] = 0x7F7F7F7F;
    const bool keep = e.keep_scratch;
    e.keep_scratch = true;
    e.overrun = false;
    unsigned long long cursor = 0;
    for (u64 c0 = 0; c0 < n64; c0 += chunk) {
        const u64 c1 = std::min<u64>(n64, c0 + chunk);
        MatchIO io;
        io.blob = text.p; io.blob_bytes = offs[c1]; io.readable_bytes = (offs[c1] + 15u) & ~15u; io.offs = offs + c0; io.n = c1 - c0;
        io.spans = out_spans + c0; io.status = status + c0; io.out = out_ids; io.cap = cap_ids;
        cursor = e.match(io, flags & 2u, c0 != 0).cursor;
    }
    e.keep_scratch = keep;
    if (e.overrun) return -60;
    *needed = cursor;
    return cursor > cap_ids ? -3 : 0;
}

void emu_set_knobs(void* h, uint32_t tile_chunk, int32_t k2_ctas, uint32_t diag_flags, uint32_t graph_cap) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    e.tile_chunk = tile_chunk; e.k2_ctas = k2_ctas; e.diag_flags = diag_flags; e.graph_cap = graph_cap;
}
// on != 0: one scratch kept across calls (a match context's); 0: a fresh, exactly sized one per call (the kept one is freed)
void emu_keep_scratch(void* h, uint32_t on) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    e.keep_scratch = on != 0;
    if (!on) for (Block* b : {&e.kept.tok, &e.kept.tok8, &e.kept.meta, &e.kept.slow, &e.kept.sort, &e.kept.hist, &e.kept.ctrl, &e.kept.gstack, &e.kept.gpool}) { b->release(); b->cap = 0; }
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
struct GatherWorld : GatherLayout {
    std::vector<std::vector<char>> store;
    std::vector<char*> block;
    std::vector<u32> epoch;
    std::vector<unsigned long long> cursor;      // the match cursor of every rank's last step (k_gather_push / k_gather_finish read it)
};
void* emu_gather_new(uint32_t world, uint64_t slab_topics, uint64_t slab_ids) {
    GatherWorld* g = new GatherWorld();
    static_cast<GatherLayout&>(*g) = gather_layout(world, slab_topics, slab_ids);
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
        const Text text(blob_in, offs[n_entries]);
        const GatherTarget target{&G, G.block.data(), rank, direct != 0};
        MatchIO io;
        io.blob = text.p; io.blob_bytes = text.bytes; io.readable_bytes = text.readable; io.offs = offs; io.sel = sel; io.n = n;
        io.cap = G.slab_ids; io.status = status; io.gather = &target;
        e.overrun = false;
        G.cursor[rank] = e.match(io, false).cursor;
        if (e.overrun) return -60;
        if (G.cursor[rank] > G.slab_ids) return -3;
    }
    if (!direct && G.world > 1)
        emu::launch(dim3(EMU_SMS * 4), dim3(256), [&] {
            k_gather_push(G.block.data(), rank, G.world, GatherLayout::off_ids, G.off_spans, G.off_index, rank * G.slab_topics, rank * G.slab_ids, n, &G.cursor[rank]);
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
    std::memcpy(ids, b + GatherLayout::off_ids, static_cast<size_t>(G.world) * G.slab_ids * 4);
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
    const Text text(blob_in, offs[nq]);
    const RetainPlan p = plan_retain(nq, rv.max_depth, cap_items, cap_desc, EMU_SMS);
    Arena a;
    RetainScratch r{};
    r.tok = a.get<u32>(p.tok); r.tok8 = a.get<u32>(p.tok8); r.meta = a.get<u32>(p.meta); r.rq = a.get<u32>(p.rq); r.ctl = a.get<RCtl>(p.ctl);
    r.front[0] = a.get<RTask>(p.front); r.front[1] = a.get<RTask>(p.front); r.descs = a.get<RDesc>(p.descs);
    std::memset(r.ctl, 0, p.ctl); std::memset(r.rq, 0, p.rq);        // what engine.cu clears before a retained lookup
    for (u32 i = 0; i < nq; ++i) status[i] = 0x7F7F7F7F;
    launch_retain(p, r, tv, rv, text.p, text.bytes, offs, out_spans, out_ids, cap_ids, status, stats_on != 0, nullptr);
    if (!a.intact()) return -60;
    RCtl& ctl = *r.ctl;
    if (work) { work[0] = ctl.stats[0]; work[1] = ctl.stats[1]; }
    if (ctl.err) return -100 - static_cast<int32_t>(ctl.err);      // scratch overflow: bit 0 tasks, bit 1 descriptors (the engine grows and retries)
    e.last_tasks.assign(p.depth + 2, 0);                           // the totals of engine.cu's `retain stats` line
    for (u32 l = 0; l <= p.depth + 1; ++l) for (u32 k = 0; k < RQ; ++k) e.last_tasks[l] += ctl.round_counts(l)[k];
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

// gm_relations_expand_device over host arrays (k_relations<false>)
int32_t emu_relations(const gm_span* spans, const uint32_t* ids, uint64_t n, const uint32_t* pubs, const gm_rel* rels, uint64_t n_rels, gm_span* out_spans,
                      gm_sub_relation* out_rels, uint64_t cap_rels, uint32_t* out_sub_ids, uint64_t cap_sub_ids, uint64_t* needed3, int32_t* status) {
    needed3[0] = needed3[1] = needed3[2] = 0;
    if (n == 0) return 0;
    launch_relations(spans, ids, n, pubs, rels, n_rels, nullptr, gm_rel_out{out_spans, out_rels, cap_rels, out_sub_ids, cap_sub_ids, needed3, status}, EMU_SMS, nullptr);
    return 0;
}

}  // extern "C"
