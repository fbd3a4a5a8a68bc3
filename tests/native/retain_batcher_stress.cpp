// Concurrency stress of the retained batcher (rmqtt_b200/csrc/retain_batcher.cpp over batcher.cpp's queue) WITHOUT a device:
// both translation units use only the public C ABI, so the entry points they reference are stubbed here.  gm_retain_match_batch
// answers every filter with handles derived from the filter's bytes, after a short sleep standing in for the device; filters
// starting with '!' are invalid.  Checked: every submitted cookie gets exactly one callback with the handles of ITS filter, from
// several producer threads, for several (max_batch, max_wait_us, dispatchers) settings; the per-filter invalid status; an
// output that outgrows the dispatcher's buffer (GM_ERR_CAPACITY protocol); a failing batch; gm_submit_publish refused; the
// PUBLISH call never reached; the probe over the same batcher.  Built with -fsanitize=thread and -fsanitize=address,undefined by
// tests/test_retain_batcher_cpu.py.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/gpumqtt.h"

static std::atomic<int> g_fail_next{0};
static std::atomic<uint64_t> g_batches{0}, g_capacity_retries{0}, g_publish_calls{0};

static uint32_t fnv(const char* s, uint32_t n) { uint32_t h = 2166136261u; for (uint32_t i = 0; i < n; ++i) h = (h ^ static_cast<unsigned char>(s[i])) * 16777619u; return h; }
static uint32_t handles_of(uint32_t h) { return h % 11 == 0 ? 5000u : h % 4; }     // a few `#`-like filters match many retained messages

extern "C" {
struct gm_engine { int dummy; };
void* gm_host_alloc_near(gm_engine*, uint64_t bytes) { return std::malloc(bytes ? bytes : 1); }
void gm_host_free(void* p) { std::free(p); }
const char* gm_last_error(gm_engine*) { return "stub"; }
// (referenced by batcher.cpp's PUBLISH batcher and churn probe; a retained batcher must never call them)
int32_t gm_sub_add(gm_engine*, const char*, uint32_t, uint32_t, int32_t*) { return GM_ERR_INTERNAL; }
int32_t gm_sub_remove(gm_engine*, const char*, uint32_t, uint32_t, int32_t*) { return GM_ERR_INTERNAL; }
int32_t gm_flush(gm_engine*) { return GM_ERR_INTERNAL; }
int32_t gm_match_batch(gm_engine*, const char*, const uint32_t*, uint64_t, gm_span*, uint32_t*, uint64_t, uint64_t*, int32_t*) {
    g_publish_calls.fetch_add(1);
    return GM_ERR_INTERNAL;
}
int32_t gm_retain_match_batch(gm_engine*, const char* blob, const uint32_t* offs, uint64_t n, gm_span* spans, uint32_t* ids, uint64_t cap, uint64_t* needed, int32_t* status) {
    g_batches.fetch_add(1);
    std::this_thread::sleep_for(std::chrono::microseconds(50));
    if (g_fail_next.exchange(0)) return GM_ERR_CUDA;
    uint64_t total = 0;
    auto invalid = [&](uint64_t i) { return offs[i + 1] > offs[i] && blob[offs[i]] == '!'; };
    for (uint64_t i = 0; i < n; ++i) if (!invalid(i)) total += handles_of(fnv(blob + offs[i], offs[i + 1] - offs[i]));
    *needed = total;
    if (total > cap) { g_capacity_retries.fetch_add(1); return GM_ERR_CAPACITY; }
    uint64_t w = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t len = offs[i + 1] - offs[i], h = fnv(blob + offs[i], len), c = invalid(i) ? 0u : handles_of(h);
        status[i] = invalid(i) ? GM_ERR_INVALID_TOPIC : GM_OK;
        spans[i] = gm_span{static_cast<uint32_t>(w), c};
        for (uint32_t k = 0; k < c; ++k) ids[w++] = h ^ (k * 2654435761u);
    }
    return GM_OK;
}
}

struct Sink {
    std::vector<std::atomic<uint32_t>> seen;
    std::vector<std::string> filters;
    std::atomic<uint64_t> bad{0}, failed{0}, invalid{0};
    explicit Sink(size_t n) : seen(n), filters(n) {}
};

static void on_match(void* user, uint64_t cookie, int32_t status, const uint32_t* ids, uint32_t n_ids) {
    Sink* s = static_cast<Sink*>(user);
    s->seen[cookie].fetch_add(1);
    const std::string& f = s->filters[cookie];
    if (status == GM_ERR_CUDA) { if (n_ids != 0) s->bad.fetch_add(1); s->failed.fetch_add(1); return; }      // the whole batch failed
    if (!f.empty() && f[0] == '!') { if (status != GM_ERR_INVALID_TOPIC || n_ids != 0) s->bad.fetch_add(1); else s->invalid.fetch_add(1); return; }
    const uint32_t h = fnv(f.data(), static_cast<uint32_t>(f.size()));
    if (status != GM_OK || n_ids != handles_of(h)) { s->bad.fetch_add(1); return; }
    for (uint32_t k = 0; k < n_ids; ++k) if (ids[k] != (h ^ (k * 2654435761u))) { s->bad.fetch_add(1); return; }
}

static int run(uint32_t max_batch, uint32_t wait_us, uint32_t dispatchers, int producers, int per_producer, bool inject_failure) {
    gm_engine eng{0};
    const size_t total = static_cast<size_t>(producers) * per_producer;
    Sink sink(total);
    for (size_t i = 0; i < total; ++i) {
        const std::string k = std::to_string(i * 2654435761u % 100003);
        sink.filters[i] = i % 89 == 0 ? "!bad/" + k : (i % 3 == 0 ? "s/" + k + "/+" : (i % 3 == 1 ? "s/" + k + "/#" : "s/" + k + "/x"));
    }
    gm_batcher_config cfg{};
    cfg.struct_size = sizeof(cfg); cfg.max_batch = max_batch; cfg.max_wait_us = wait_us; cfg.dispatchers = dispatchers; cfg.on_match = on_match; cfg.user = &sink;
    gm_batcher* b = nullptr;
    if (gm_retain_batcher_create(&eng, &cfg, &b) != GM_OK) return 1;
    // a PUBLISH packet is not a filter: refused, and nothing is queued
    const uint8_t pkt[] = {0x30, 0x05, 0x00, 0x03, 'a', '/', 'b'};
    const bool publish_refused = gm_submit_publish(b, pkt, sizeof(pkt), 0) == GM_ERR_INVALID_ARG;
    if (inject_failure) g_fail_next.store(1);
    std::vector<std::thread> th;
    for (int p = 0; p < producers; ++p)
        th.emplace_back([&, p] {
            for (int i = 0; i < per_producer; ++i) {
                const size_t c = static_cast<size_t>(p) * per_producer + i;
                if (gm_submit(b, sink.filters[c].data(), static_cast<uint32_t>(sink.filters[c].size()), c) != GM_OK) std::abort();
                if (i % 1000 == 999) gm_batcher_drain(b);
            }
        });
    for (auto& t : th) t.join();
    gm_batcher_drain(b);
    size_t once = 0;
    for (size_t i = 0; i < total; ++i) once += sink.seen[i].load() == 1;
    gm_batcher_destroy(b);
    const bool ok = publish_refused && once == total && sink.bad.load() == 0 && sink.invalid.load() > 0 &&
                    (inject_failure ? sink.failed.load() > 0 : sink.failed.load() == 0);
    printf("retained batcher max_batch %u wait %u us dispatchers %u producers %d: %zu/%zu delivered once, bad %llu, invalid %llu, failed %llu, publish refused %d -> %s\n",
           max_batch, wait_us, dispatchers, producers, once, total, (unsigned long long)sink.bad.load(), (unsigned long long)sink.invalid.load(),
           (unsigned long long)sink.failed.load(), publish_refused ? 1 : 0, ok ? "ok:" : "FAILED");
    return ok ? 0 : 1;
}

// the destroy of a batcher with work still queued delivers it first
static int destroy_drains() {
    gm_engine eng{0};
    Sink sink(300);
    for (size_t i = 0; i < 300; ++i) sink.filters[i] = "d/" + std::to_string(i) + "/+";
    gm_batcher_config cfg{};
    cfg.struct_size = sizeof(cfg); cfg.max_batch = 4096; cfg.max_wait_us = 100000; cfg.dispatchers = 2; cfg.on_match = on_match; cfg.user = &sink;
    gm_batcher* b = nullptr;
    if (gm_retain_batcher_create(&eng, &cfg, &b) != GM_OK) return 1;
    for (size_t i = 0; i < 300; ++i) gm_submit(b, sink.filters[i].data(), static_cast<uint32_t>(sink.filters[i].size()), i);
    gm_batcher_destroy(b);
    size_t once = 0;
    for (size_t i = 0; i < 300; ++i) once += sink.seen[i].load() == 1;
    const bool ok = once == 300 && sink.bad.load() == 0;
    printf("retained batcher destroy with 300 queued: %zu delivered once -> %s\n", once, ok ? "ok:" : "FAILED");
    return ok ? 0 : 1;
}

static int probe() {
    gm_engine eng{0};
    std::string blob;
    std::vector<uint32_t> offs{0u};
    double want = 0;
    for (int i = 0; i < 40; ++i) { const std::string f = "p/" + std::to_string(i) + "/+"; blob += f; offs.push_back(static_cast<uint32_t>(blob.size())); want += handles_of(fnv(f.data(), static_cast<uint32_t>(f.size()))); }
    gm_latency lat{};
    const int32_t rc = gm_retain_batcher_probe(&eng, blob.data(), offs.data(), 40, 8, 25, 0, &lat);
    const bool ok = rc == GM_OK && lat.samples == 200 && lat.p50_us > 0 && lat.p50_us <= lat.p99_us && lat.p99_us <= lat.max_us && lat.topics_per_s > 0 &&
                    lat.ids_per_topic == want / 40;
    printf("retained probe burst 8 x 25: rc %d samples %llu ids/filter %.2f (want %.2f) -> %s\n", rc, (unsigned long long)lat.samples, lat.ids_per_topic, want / 40, ok ? "ok:" : "FAILED");
    return ok ? 0 : 1;
}

int main() {
    int rc = 0;
    rc |= run(1, 0, 1, 1, 2000, false);
    rc |= run(64, 200, 2, 4, 5000, false);
    rc |= run(4096, 500, 3, 6, 8000, false);          // big batches: the handle list outgrows the dispatcher's first buffer
    rc |= run(256, 100, 2, 3, 3000, true);            // one failing batch: its filters get the error, the rest are served
    rc |= destroy_drains();
    rc |= probe();
    const bool retried = g_capacity_retries.load() > 0, no_publish = g_publish_calls.load() == 0;
    printf("batches %llu, capacity retries %llu, PUBLISH calls %llu -> %s\n", (unsigned long long)g_batches.load(), (unsigned long long)g_capacity_retries.load(),
           (unsigned long long)g_publish_calls.load(), retried && no_publish ? "ok:" : "FAILED");
    return rc | (retried && no_publish ? 0 : 1);
}
