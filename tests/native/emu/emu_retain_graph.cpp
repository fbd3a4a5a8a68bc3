// TEST INFRASTRUCTURE: the small-graph form of the retained lookup (engine.cu small_graph_retain) over HOST memory, on the CPU
// emulation in cuda_runtime.h.  It extends emu_driver.cpp — whose engine, device image, poisoned scratch and guarded text it
// needs — by including that translation unit, so the library built from this file exports the whole driver plus
// emu_retain_match_graph.  Exposed as a small C interface for tests/test_emu_retain_graph.py.  Build (the test does it):
//   g++ -O1 -g -std=c++17 -DGM_CPU_EMU -Itests/native/emu -Irmqtt_b200/csrc -shared -fPIC tests/native/emu/emu_retain_graph.cpp \
//       rmqtt_b200/csrc/host_trie.cpp rmqtt_b200/csrc/retain_tree.cpp -o <out>.so     (+ -fsanitize=address,undefined for the ASan run)
#include "emu_driver.cpp"

extern "C" {

// RetainStorage::get for a batch of filters, launched as the captured graph launches it: the kernels are sized for a CAPACITY
// of `rows` filters (0: the batch size + 37) and read the real count and text length from a header in memory.  Rows past the
// batch are poisoned: their offsets are garbage, their status / span slots hold a pattern that must survive (-50 / -51), and
// their token rows hold a stale, valid filter `#`, as the scratch of an earlier, larger batch would.  Returns as
// emu_retain_match (0, -3 with *needed, -100 - overflow bits, -60), and -2 when rows < n.  emu_retain_last_tasks then reports
// this lookup's tasks per round.
int32_t emu_retain_match_graph(void* h, const char* blob_in, const uint32_t* offs, uint64_t n64, uint32_t rows, uint32_t stats_on, uint32_t cap_items,
                               uint32_t cap_desc, gm_span* out_spans, uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed, int32_t* status, uint64_t* work) {
    EmuEngine& e = *static_cast<EmuEngine*>(h);
    const u32 nq = static_cast<u32>(n64);
    *needed = 0;
    if (nq == 0) return 0;
    const u32 n = rows ? rows : nq + 37u;                            // launch size
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
    std::memset(r.ctl, 0, p.ctl); std::memset(r.rq, 0, p.rq);        // what engine.cu clears before a retained lookup
    const u32 hdr[4] = {nq, text.bytes, 0u, 0u};
    std::vector<u32> offs_cap(offs, offs + nq + 1);                  // the in-block holds capacity + 1 offsets; the tail is never read
    offs_cap.resize(static_cast<size_t>(n) + 1, 0xDEADBEEFu);
    std::vector<int32_t> status_cap(n, 0x7F7F7F7F);
    std::vector<gm_span> spans_cap(n, gm_span{0xABABABABu, 0xABABABABu});
    for (u32 q = nq; q < n; ++q) { r.meta[q] = 1u; r.tok8[static_cast<size_t>(q) * TOK8] = TOK_HASH; }
    launch_retain(p, r, tv, rv, text.p, text.bytes, offs_cap.data(), spans_cap.data(), out_ids, cap_ids, status_cap.data(), stats_on != 0, nullptr, hdr);
    if (!a.intact()) return -60;
    for (u32 i = nq; i < n; ++i) if (status_cap[i] != 0x7F7F7F7F) return -50;      // a row beyond the real batch was touched
    for (u32 i = nq; i < n; ++i) if (spans_cap[i].off != 0xABABABABu || spans_cap[i].cnt != 0xABABABABu) return -51;
    std::memcpy(status, status_cap.data(), nq * sizeof(int32_t));
    std::memcpy(out_spans, spans_cap.data(), nq * sizeof(gm_span));
    RCtl& ctl = *r.ctl;
    if (work) { work[0] = ctl.stats[0]; work[1] = ctl.stats[1]; }
    if (ctl.err) return -100 - static_cast<int32_t>(ctl.err);      // scratch overflow: bit 0 tasks, bit 1 descriptors (the engine grows and retries)
    e.last_tasks.assign(p.depth + 2, 0);
    for (u32 l = 0; l <= p.depth + 1; ++l) for (u32 k = 0; k < RQ; ++k) e.last_tasks[l] += ctl.round_counts(l)[k];
    e.last_n_desc = 0;
    for (u32 k = 0; k < RQ; ++k) e.last_n_desc += ctl.n_desc[k];
    *needed = ctl.grand;
    return ctl.grand > cap_ids ? -3 : 0;
}

}  // extern "C"
