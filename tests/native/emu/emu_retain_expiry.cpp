// TEST INFRASTRUCTURE: retained lookups with deadlines (gm_retain_match_batch_at) over HOST memory, on the CPU emulation in
// cuda_runtime.h.  It extends emu_retain_graph.cpp (and through it emu_driver.cpp: engine, poisoned scratch, guarded text) by
// including that translation unit, and adds the deadline calls and a lookup that hands launch_retain the host tree's deadline
// table and a `now` in memory, in the pipelined form or in the small-graph form (capacity rows, header in memory).  Exposed as
// a small C interface for tests/test_retain_expiry_cpu.py.  Build (the test does it):
//   g++ -O1 -g -std=c++17 -DGM_CPU_EMU -Itests/native/emu -Irmqtt_b200/csrc -shared -fPIC tests/native/emu/emu_retain_expiry.cpp \
//       rmqtt_b200/csrc/host_trie.cpp rmqtt_b200/csrc/retain_tree.cpp -o <out>.so     (+ -fsanitize=address,undefined for the ASan run)
#include "emu_retain_graph.cpp"

extern "C" {

int32_t emu_retain_set_ttl(void* h, const char* t, uint32_t len, uint32_t value, uint64_t deadline) {
    return static_cast<EmuEngine*>(h)->rtree.set_ttl(t, len, value, deadline, nullptr, nullptr);
}
uint64_t emu_retain_bulk_load_ttl(void* h, const char* blob, const uint32_t* offs, const uint32_t* vals, const uint64_t* dl, uint64_t n) {
    return static_cast<EmuEngine*>(h)->rtree.set_batch_ttl(blob, offs, vals, dl, n);
}
uint64_t emu_retain_remove_expired(void* h, uint64_t now, uint32_t* out, uint64_t cap) { return static_cast<EmuEngine*>(h)->rtree.remove_expired(now, out, cap); }

// RetainStorage::get at `now` for a batch of filters.  rows == 0: the pipelined form; else the small-graph form launched for a
// capacity of `rows` filters, rows past the batch poisoned as in emu_retain_match_graph (-50 / -51 when one was touched).
// Returns as emu_retain_match.
int32_t emu_retain_match_at(void* h, uint64_t now, const char* blob_in, const uint32_t* offs, uint64_t n64, uint32_t rows, uint32_t cap_items, uint32_t cap_desc,
                            gm_span* out_spans, uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed, int32_t* status) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    const u32 nq = static_cast<u32>(n64);
    *needed = 0;
    if (nq == 0) return 0;
    const u32 n = rows ? rows : nq;
    if (n < nq) return -2;
    if (!e.prepare(true)) return -7;
    const TrieView tv = e.view();
    const RetainView rv = e.rview();
    const Text text(blob_in, offs[nq]);
    const RetainPlan p = plan_retain(n, rv.max_depth, cap_items, cap_desc, EMU_SMS);
    Arena a;
    RetainScratch r{};
    r.tok = a.get<u32>(p.tok); r.tok8 = a.get<u32>(p.tok8); r.meta = a.get<u32>(p.meta); r.rq = a.get<u32>(p.rq); r.ctl = a.get<RCtl>(p.ctl);
    r.front[0] = a.get<RTask>(p.front); r.front[1] = a.get<RTask>(p.front); r.descs = a.get<RDesc>(p.descs);
    std::memset(r.ctl, 0, p.ctl); std::memset(r.rq, 0, p.rq);
    u32 hdr[4] = {nq, text.bytes, 0u, 0u};
    std::memcpy(hdr + 2, &now, sizeof(now));
    u64* now_mem = a.get<u64>(sizeof(u64));
    *now_mem = now;
    RetainDeadlines x;
    if (const u32 nd = e.rtree.dl_lookup_size()) { x.dl = e.rtree.dl.data(); x.n = nd; x.now = rows ? reinterpret_cast<const u64*>(hdr + 2) : now_mem; }
    std::vector<u32> offs_cap(offs, offs + nq + 1);
    offs_cap.resize(static_cast<size_t>(n) + 1, 0xDEADBEEFu);
    std::vector<int32_t> status_cap(n, 0x7F7F7F7F);
    std::vector<gm_span> spans_cap(n, gm_span{0xABABABABu, 0xABABABABu});
    if (rows) for (u32 q = nq; q < n; ++q) { r.meta[q] = 1u; r.tok8[static_cast<size_t>(q) * TOK8] = TOK_HASH; }
    launch_retain(p, r, tv, rv, text.p, text.bytes, rows ? offs_cap.data() : offs, spans_cap.data(), out_ids, cap_ids, status_cap.data(), false, nullptr,
                  rows ? hdr : nullptr, x);
    if (!a.intact()) return -60;
    for (u32 i = nq; i < n; ++i) if (status_cap[i] != 0x7F7F7F7F) return -50;
    for (u32 i = nq; i < n; ++i) if (spans_cap[i].off != 0xABABABABu || spans_cap[i].cnt != 0xABABABABu) return -51;
    std::memcpy(status, status_cap.data(), nq * sizeof(int32_t));
    std::memcpy(out_spans, spans_cap.data(), nq * sizeof(gm_span));
    RCtl& ctl = *r.ctl;
    if (ctl.err) return -100 - static_cast<int32_t>(ctl.err);
    *needed = ctl.grand;
    return ctl.grand > cap_ids ? -3 : 0;
}

}  // extern "C"
