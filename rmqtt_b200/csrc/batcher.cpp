// Single-call front end of libgpumqtt: the MPSC micro-batcher (SURVEY.md §8(b), Threading row).
//
// The reference calls Router::matches ONCE PER PUBLISH from many tokio worker threads
// (rmqtt/src/router.rs:482-484, caller rmqtt/src/shared.rs:601-636).  A GPU wants batches.  The batcher sits between
// the two: gm_submit() appends one topic to a queue (a mutex-protected append, never touches the device) and
// dispatch threads turn the queue into gm_match_batch() calls — when `max_batch` topics are queued or the oldest one
// has waited `max_wait_us`.  With two (or more) dispatchers one batch is being collected while another is on the
// device; the engine keeps several batches in flight (match contexts, engine.cu) and serves small ones as a single
// CUDA-graph launch.  Results come back through a callback per topic (a Rust caller completes a oneshot / writes an
// eventfd there).  Only the public C ABI is used here.  The same queue serves the retained lookup (retain_batcher.cpp): a
// batcher holds the engine call it dispatches to (batcher_internal.h).
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "batcher_internal.h"

namespace {
using Clock = std::chrono::steady_clock;

struct Pending {
    std::vector<char> blob;
    std::vector<uint32_t> offs{0u};
    std::vector<uint64_t> cookies;
    Clock::time_point first;
    void clear() { blob.clear(); offs.assign(1, 0u); cookies.clear(); }
    size_t count() const { return cookies.size(); }
};
}  // namespace

struct gm_batcher {
    gm_engine* e = nullptr;
    gm::BatcherTarget target{};
    gm_batcher_config cfg{};
    std::mutex mu;
    std::condition_variable cv_work, cv_drain;
    Pending pending;
    uint64_t submitted = 0, delivered = 0;
    bool stop = false;
    std::vector<std::thread> threads;

    void run() {
        Pending local;
        std::vector<gm_span> spans;
        std::vector<int32_t> status;
        uint32_t* ids = nullptr;
        uint64_t ids_cap = 0;
        auto grow_ids = [&](uint64_t want) {
            if (want <= ids_cap) return true;
            uint64_t ncap = std::max<uint64_t>(want, ids_cap * 2 + 4096);
            uint32_t* np = static_cast<uint32_t*>(gm_host_alloc_near(e, ncap * sizeof(uint32_t)));
            if (!np) return false;
            if (ids) gm_host_free(ids);
            ids = np; ids_cap = ncap;
            return true;
        };
        grow_ids(1 << 16);
        std::unique_lock<std::mutex> lk(mu);
        for (;;) {
            cv_work.wait(lk, [&] { return stop || pending.count() > 0; });
            if (pending.count() == 0) { if (stop) break; continue; }
            // the window: dispatch when the batch is full or its oldest topic has waited long enough
            while (!stop && pending.count() < cfg.max_batch) {
                const auto deadline = pending.first + std::chrono::microseconds(cfg.max_wait_us);
                if (Clock::now() >= deadline) break;
                cv_work.wait_until(lk, deadline);
                if (pending.count() == 0) break;          // another dispatcher took it
            }
            if (pending.count() == 0) continue;
            std::swap(local, pending);
            pending.clear();
            lk.unlock();

            const uint64_t n = local.count();
            spans.resize(n); status.resize(n);
            uint64_t needed = 0;
            int32_t rc;
            for (;;) {
                rc = target.call(e, local.blob.data(), local.offs.data(), n, spans.data(), ids, ids_cap, &needed, status.data());
                if (rc != GM_ERR_CAPACITY || !grow_ids(needed)) break;
            }
            if (rc != GM_OK) {                      // the whole batch failed: every topic gets the error; say why (first few times)
                static std::atomic<int> shown{0};
                if (shown.fetch_add(1) < 5) fprintf(stderr, "libgpumqtt batcher: %s(%llu topics) failed with %d: %s\n", target.name, (unsigned long long)n, rc, gm_last_error(e));
            }
            for (uint64_t i = 0; i < n; ++i) {
                const int32_t st = rc == GM_OK ? status[i] : rc;
                cfg.on_match(cfg.user, local.cookies[i], st, (rc == GM_OK && st == GM_OK) ? ids + spans[i].off : nullptr, (rc == GM_OK && st == GM_OK) ? spans[i].cnt : 0u);
            }
            local.clear();
            lk.lock();
            delivered += n;
            cv_drain.notify_all();
        }
        lk.unlock();
        if (ids) gm_host_free(ids);
    }
};

namespace {
const gm::BatcherTarget kPublish{gm_match_batch, "gm_match_batch", true};
}

int32_t gm::batcher_create(gm_engine* e, const gm_batcher_config* cfg, const BatcherTarget& target, gm_batcher** out) {
    if (!e || !cfg || !out || !cfg->on_match) return GM_ERR_INVALID_ARG;
    gm_batcher* b = new gm_batcher();
    b->e = e;
    b->target = target;
    std::memcpy(&b->cfg, cfg, std::min<size_t>(cfg->struct_size ? cfg->struct_size : sizeof(gm_batcher_config), sizeof(gm_batcher_config)));
    if (b->cfg.max_batch == 0) b->cfg.max_batch = 4096;
    if (b->cfg.dispatchers == 0) b->cfg.dispatchers = 2;
    b->cfg.dispatchers = std::min<uint32_t>(b->cfg.dispatchers, 8);
    for (uint32_t i = 0; i < b->cfg.dispatchers; ++i) b->threads.emplace_back([b] { b->run(); });
    *out = b;
    return GM_OK;
}

extern "C" {

int32_t gm_batcher_create(gm_engine* e, const gm_batcher_config* cfg, gm_batcher** out) { return gm::batcher_create(e, cfg, kPublish, out); }

int32_t gm_submit(gm_batcher* b, const char* topic, uint32_t len, uint64_t cookie) {
    if (!b || (!topic && len)) return GM_ERR_INVALID_ARG;
    bool wake;
    {
        std::lock_guard<std::mutex> g(b->mu);
        Pending& p = b->pending;
        if (p.blob.size() + len > 0xFFFF0000ull) return GM_ERR_TOO_LARGE;
        if (p.count() == 0) p.first = Clock::now();
        p.blob.insert(p.blob.end(), topic, topic + len);
        p.offs.push_back(static_cast<uint32_t>(p.blob.size()));
        p.cookies.push_back(cookie);
        b->submitted++;
        wake = p.count() == 1 || p.count() == b->cfg.max_batch;     // a dispatcher sleeps only on an empty queue or inside the window
    }
    if (wake) b->cv_work.notify_one();
    return GM_OK;
}

// ---- wire-side batching (SURVEY §8f-4): the topic of a raw PUBLISH packet goes straight into the batch ----------------
// MQTT 3.1.1 and 5 share the layout: fixed header (type 3 << 4 | flags), remaining-length varint (<= 4 bytes), then the
// topic name as a u16-big-endian-prefixed string — the first field both decoders read
// (rmqtt-codec/src/v3/decode.rs:103-104, rmqtt-codec/src/v5/packet/publish.rs:27-28; varint: rmqtt-codec/src/utils.rs:142-155).
int32_t gm_publish_topic(const uint8_t* packet, uint32_t len, const char** topic, uint32_t* topic_len) {
    if (!packet || !topic || !topic_len || len < 2) return GM_ERR_INVALID_ARG;
    if ((packet[0] >> 4) != 3) return GM_ERR_INVALID_ARG;                 // not a PUBLISH
    uint32_t pos = 1, rem = 0, shift = 0;
    for (;;) {
        if (pos >= len) return GM_ERR_INVALID_ARG;                        // MalformedPacket
        const uint8_t v = packet[pos++];
        rem += static_cast<uint32_t>(v & 0x7F) << shift;
        if (!(v & 0x80)) break;
        if (shift >= 21) return GM_ERR_INVALID_ARG;                       // InvalidLength
        shift += 7;
    }
    if (rem < 2 || pos + 2 > len) return GM_ERR_INVALID_ARG;
    const uint32_t tl = (static_cast<uint32_t>(packet[pos]) << 8) | packet[pos + 1];
    pos += 2;
    if (tl + 2 > rem || pos + tl > len) return GM_ERR_INVALID_ARG;
    *topic = reinterpret_cast<const char*>(packet + pos);
    *topic_len = tl;
    return GM_OK;
}

int32_t gm_submit_publish(gm_batcher* b, const uint8_t* packet, uint32_t len, uint64_t cookie) {
    if (b && !b->target.raw_packets) return GM_ERR_INVALID_ARG;        // a retained batcher takes filters, not PUBLISH topics
    const char* t = nullptr;
    uint32_t tl = 0;
    const int32_t rc = gm_publish_topic(packet, len, &t, &tl);
    return rc == GM_OK ? gm_submit(b, t, tl, cookie) : rc;
}

int32_t gm_batcher_drain(gm_batcher* b) {
    if (!b) return GM_ERR_INVALID_ARG;
    std::unique_lock<std::mutex> lk(b->mu);
    const uint64_t target = b->submitted;
    b->cv_drain.wait(lk, [&] { return b->delivered >= target; });
    return GM_OK;
}

void gm_batcher_destroy(gm_batcher* b) {
    if (!b) return;
    gm_batcher_drain(b);
    { std::lock_guard<std::mutex> g(b->mu); b->stop = true; }
    b->cv_work.notify_all();
    for (auto& t : b->threads) t.join();
    delete b;
}

}  // extern "C"

// ---- closed-loop latency probe ------------------------------------------------------------------------------------
namespace {
struct Probe {
    std::vector<Clock::time_point> t_submit;
    std::vector<float> lat_us;
    std::atomic<uint64_t> done{0};
    std::atomic<uint64_t> ids{0};
};
void probe_cb(void* user, uint64_t cookie, int32_t, const uint32_t*, uint32_t n_ids) {
    Probe* p = static_cast<Probe*>(user);
    p->lat_us[cookie] = std::chrono::duration<float, std::micro>(Clock::now() - p->t_submit[cookie]).count();
    p->ids.fetch_add(n_ids, std::memory_order_relaxed);
    p->done.fetch_add(1, std::memory_order_release);
}
}  // namespace

int32_t gm::batcher_probe(gm_engine* e, const BatcherTarget& target, const char* blob, const uint32_t* offsets, uint64_t n, uint32_t burst, uint32_t rounds,
                          uint32_t max_wait_us, gm_latency* out) {
    if (!e || !blob || !offsets || !out || n == 0 || burst == 0 || rounds == 0) return GM_ERR_INVALID_ARG;
    Probe p;
    const uint64_t total = static_cast<uint64_t>(burst) * rounds;
    p.t_submit.resize(total);
    p.lat_us.assign(total, 0.f);
    gm_batcher_config cfg{};
    cfg.struct_size = sizeof(cfg); cfg.max_batch = burst; cfg.max_wait_us = max_wait_us; cfg.dispatchers = 2; cfg.on_match = probe_cb; cfg.user = &p;
    gm_batcher* b = nullptr;
    int32_t rc = gm::batcher_create(e, &cfg, target, &b);
    if (rc != GM_OK) return rc;
    // warm-up round (graph capture, scratch allocation) — not measured
    {
        for (uint32_t i = 0; i < burst; ++i) { const uint64_t t = i % n; p.t_submit[i] = Clock::now(); gm_submit(b, blob + offsets[t], offsets[t + 1] - offsets[t], i); }
        gm_batcher_drain(b);
        p.done.store(0); p.ids.store(0);
    }
    const auto t0 = Clock::now();
    uint64_t k = 0, cursor = burst;        // topics cycle through the provided batch
    for (uint32_t r = 0; r < rounds; ++r) {
        const uint64_t want = k + burst;
        for (uint32_t i = 0; i < burst; ++i, ++k, ++cursor) {
            const uint64_t t = cursor % n;
            p.t_submit[k] = Clock::now();
            gm_submit(b, blob + offsets[t], offsets[t + 1] - offsets[t], k);
        }
        while (p.done.load(std::memory_order_acquire) < want) {      // closed loop: the next burst is offered when this one is answered
            if (burst >= 1024) std::this_thread::yield();
        }
    }
    const double secs = std::chrono::duration<double>(Clock::now() - t0).count();
    gm_batcher_destroy(b);
    std::vector<float> v = p.lat_us;
    std::sort(v.begin(), v.end());
    double sum = 0;
    for (float x : v) sum += x;
    out->samples = total;
    out->p50_us = v[total / 2];
    out->p99_us = v[std::min<uint64_t>(total - 1, (total * 99) / 100)];
    out->mean_us = sum / total;
    out->max_us = v.back();
    out->topics_per_s = total / secs;
    out->ids_per_topic = static_cast<double>(p.ids.load()) / total;
    return GM_OK;
}

extern "C" {

int32_t gm_batcher_probe(gm_engine* e, const char* blob, const uint32_t* offsets, uint64_t n, uint32_t burst, uint32_t rounds, uint32_t max_wait_us,
                         gm_latency* out) {
    return gm::batcher_probe(e, kPublish, blob, offsets, n, burst, rounds, max_wait_us, out);
}

// ---- churn probe: subscribe / unsubscribe load against a running engine --------------------------------------------
// Cycles over the given (filter, value) pairs: Router::remove then Router::add of the same pair (rmqtt/src/router.rs:417-479),
// at `target_ops_per_s` (0 = as fast as one thread can), calling gm_flush every `flush_period_us` (0 = never: auto-flush
// engines ship pending mutations with the next match).  Meant to run in its own thread while other threads match.
int32_t gm_churn_probe(gm_engine* e, const char* blob, const uint32_t* offsets, const uint32_t* values, uint64_t n, double target_ops_per_s,
                       uint32_t duration_ms, uint32_t flush_period_us, gm_churn* out) {
    if (!e || !blob || !offsets || !values || !out || n == 0) return GM_ERR_INVALID_ARG;
    std::memset(out, 0, sizeof(*out));
    const auto t0 = Clock::now();
    const auto t_end = t0 + std::chrono::milliseconds(duration_ms);
    auto next_flush = t0 + std::chrono::microseconds(flush_period_us);
    uint64_t ops = 0, flushes = 0, i = 0;
    double flush_us_sum = 0, flush_us_max = 0;
    for (;;) {
        for (int k = 0; k < 64; ++k, i = (i + 1) % n) {
            int32_t ch = 0;
            const char* f = blob + offsets[i];
            const uint32_t len = offsets[i + 1] - offsets[i];
            int32_t rc = gm_sub_remove(e, f, len, values[i], &ch);
            if (rc == GM_OK) rc = gm_sub_add(e, f, len, values[i], &ch);
            if (rc != GM_OK) return rc;
            ops += 2;
        }
        const auto now = Clock::now();
        if (flush_period_us && now >= next_flush) {
            const int32_t rc = gm_flush(e);
            if (rc != GM_OK) return rc;
            const double us = std::chrono::duration<double, std::micro>(Clock::now() - now).count();
            flush_us_sum += us; flush_us_max = std::max(flush_us_max, us); ++flushes;
            next_flush = Clock::now() + std::chrono::microseconds(flush_period_us);
        }
        if (now >= t_end) break;
        if (target_ops_per_s > 0) {
            const double ahead = ops / target_ops_per_s - std::chrono::duration<double>(now - t0).count();
            if (ahead > 50e-6) std::this_thread::sleep_for(std::chrono::duration<double>(std::min(ahead, 2e-3)));
        }
    }
    const double secs = std::chrono::duration<double>(Clock::now() - t0).count();
    out->seconds = secs; out->ops = ops; out->flushes = flushes; out->ops_per_s = ops / secs; out->flushes_per_s = flushes / secs;
    out->mean_flush_us = flushes ? flush_us_sum / flushes : 0; out->max_flush_us = flush_us_max;
    return GM_OK;
}

}  // extern "C"
