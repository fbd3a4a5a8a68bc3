// TEST INFRASTRUCTURE: the message store (rmqtt_b200/csrc/msgstore.cuh: MsCore, its kernels and launches) over HOST memory, on
// the CPU emulation in cuda_runtime.h.  The store's host logic is the product's own; this backend gives it poisoned scratch with
// guard bytes (emu_driver.cpp's Block) and runs its retained lookup as emu_retain_expiry.cpp does, on the emulated engine.
// Exposed as a small C interface for tests/test_msgstore_cpu.py.  Build (the test does it):
//   g++ -O1 -g -std=c++17 -DGM_CPU_EMU -Itests/native/emu -Irmqtt_b200/csrc -shared -fPIC tests/native/emu/emu_msgstore.cpp \
//       rmqtt_b200/csrc/host_trie.cpp rmqtt_b200/csrc/retain_tree.cpp -o <out>.so     (+ -fsanitize=address,undefined for the ASan run)
#include "emu_retain_expiry.cpp"

#include <string>

#include "msgstore.cuh"

thread_local std::string gm::g_err;

namespace {

int map_tree(int st) {
    if (st == PARSE_OK) return GM_OK;
    if (st == RetainTreeHost::SET_CONFLICT || st == RetainTreeHost::SET_HANDLE_RANGE) return GM_ERR_INVALID_ARG;
    return st == PARSE_TOO_DEEP ? GM_ERR_TOO_DEEP : GM_ERR_INVALID_TOPIC;
}

struct EmuBackend {
    EmuEngine eng;
    u32 cap_items = 64, cap_desc = 64;       // small: the lookup's overflow-and-retry runs too
    bool overrun = false;                    // a launch wrote past a scratch block of the lookup
    std::vector<Block*> bufs;                // every Buf of the store, for the guard check
    struct Buf {
        Block b;
        void* p = nullptr;
        int ensure(size_t bytes) { p = b.get<u8>(std::max<size_t>(bytes, 1), false); return GM_OK; }
    };
    bool device() const { return true; }
    cudaStream_t stream() const { return nullptr; }
    int h2d(void* d, const void* h, size_t n) { std::memcpy(d, h, n); return GM_OK; }
    int d2h(void* h, const void* d, size_t n) { std::memcpy(h, d, n); return GM_OK; }
    int fill(void* d, int v, size_t n) { std::memset(d, v, n); return GM_OK; }
    int sync() { return GM_OK; }
    int launched() { return GM_OK; }
    int walk(u64 now, const void* blob, u64 bytes, const u32* offs, u64 n, gm_span* spans, u32* ids, u64 cap, u64* needed, int32_t* status) {
        if (!eng.prepare(true)) return GM_ERR_TOO_LARGE;
        for (;;) {
            const TrieView tv = eng.view();
            const RetainView rv = eng.rview();
            const RetainPlan p = plan_retain(static_cast<u32>(n), rv.max_depth, cap_items, cap_desc, EMU_SMS);
            Arena a;
            RetainScratch r{};
            r.tok = a.get<u32>(p.tok); r.tok8 = a.get<u32>(p.tok8); r.meta = a.get<u32>(p.meta); r.rq = a.get<u32>(p.rq); r.ctl = a.get<RCtl>(p.ctl);
            r.front[0] = a.get<RTask>(p.front); r.front[1] = a.get<RTask>(p.front); r.descs = a.get<RDesc>(p.descs);
            std::memset(r.ctl, 0, p.ctl); std::memset(r.rq, 0, p.rq);
            u64* now_mem = a.get<u64>(sizeof(u64));
            *now_mem = now;
            RetainDeadlines x;
            if (const u32 nd = eng.rtree.dl_lookup_size()) { x.dl = eng.rtree.dl.data(); x.n = nd; x.now = now_mem; }
            launch_retain(p, r, tv, rv, blob, bytes, offs, spans, ids, cap, status, false, nullptr, nullptr, x);
            if (!a.intact()) { overrun = true; return GM_ERR_INTERNAL; }
            if (r.ctl->err) { cap_items *= 4; cap_desc *= 4; continue; }
            *needed = r.ctl->grand;
            return r.ctl->grand > cap ? GM_ERR_CAPACITY : GM_OK;
        }
    }
    int set_ttl(const char* key, u32 len, u32 handle, u64 deadline) { return map_tree(eng.rtree.set_ttl(key, len, handle, deadline, nullptr, nullptr)); }
    int bulk_ttl(const char* blob, const u32* offs, const u32* handles, const u64* deadlines, u64 n, u64* n_set) {
        GM_TRY(map_tree(eng.rtree.check_batch(blob, offs, handles, deadlines, n)));
        *n_set = eng.rtree.set_batch_ttl(blob, offs, handles, deadlines, n);
        return GM_OK;
    }
    int remove_batch(const char* blob, const u32* offs, u64 n) {
        for (u64 i = 0; i < n; ++i) eng.rtree.remove(blob + offs[i], offs[i + 1] - offs[i], nullptr, nullptr);
        return GM_OK;
    }
    int remove_expired(u64 now, u32* out, u64 cap, u64* n) { *n = eng.rtree.remove_expired(now, out, cap); return GM_OK; }
};

using EmuStore = MsCore<EmuBackend>;

bool store_intact(const EmuStore& s) {
    for (const auto* b : {&s.tbl[0], &s.tbl[1], &s.d_count, &s.d_pending, &s.d_retired, &s.d_blob, &s.d_offs, &s.d_clients, &s.d_shares, &s.d_contested, &s.d_rspans,
                          &s.d_status, &s.d_raw, &s.d_owner, &s.d_keep, &s.d_cnt, &s.d_base, &s.d_cur, &s.d_cand, &s.d_state, &s.d_ckeys, &s.d_cclaim, &s.d_ctaken,
                          &s.d_cslot, &s.d_spans, &s.d_out, &s.d_ctl})
        if (!b->b.intact()) return false;
    return !s.be.overrun;
}

}  // namespace

extern "C" {

void* emu_ms_new(uint32_t initial_mark_slots) {
    auto* s = new EmuStore();
    s->num_sms = EMU_SMS;
    if (initial_mark_slots) s->init_slots = initial_mark_slots;
    return s;
}
void emu_ms_free(void* h) { delete static_cast<EmuStore*>(h); }
const char* emu_ms_error() { return g_err.c_str(); }

int32_t emu_ms_store(void* h, const char* topic, uint32_t len, uint32_t handle, uint64_t expiry, const uint32_t* clients, const uint32_t* shares, uint32_t n) {
    return static_cast<EmuStore*>(h)->store(topic, len, handle, expiry, clients, shares, n);
}
int32_t emu_ms_store_batch(void* h, const char* blob, const uint32_t* offs, const uint32_t* handles, const uint64_t* expiry, uint64_t n, const uint32_t* mark_offs,
                           const uint32_t* clients, const uint32_t* shares) {
    return static_cast<EmuStore*>(h)->store_batch(blob, offs, handles, expiry, n, mark_offs, clients, shares);
}
// as gm_msgstore_get_batch; -60 when a launch wrote past a scratch block
int32_t emu_ms_get_batch(void* h, uint64_t now, const char* blob, const uint32_t* offs, uint64_t n, const uint32_t* clients, const uint32_t* shares, gm_span* spans,
                         uint32_t* out, uint64_t cap, uint64_t* needed, int32_t* status) {
    EmuStore& s = *static_cast<EmuStore*>(h);
    const int32_t st = s.get_batch(now, blob, offs, n, clients, shares, spans, out, cap, needed, status);
    return store_intact(s) ? st : -60;
}
int32_t emu_ms_remove_expired(void* h, uint64_t now, uint32_t* out, uint64_t cap, uint64_t* n) { return static_cast<EmuStore*>(h)->remove_expired(now, out, cap, n); }
int32_t emu_ms_stats(void* h, gm_msgstore_stats* out) { return static_cast<EmuStore*>(h)->stats(out); }

}  // extern "C"
