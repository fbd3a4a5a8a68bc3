// The message store (gm_msgstore_*): rmqtt-message-storage's RAM backend (rmqtt-plugins/rmqtt-message-storage/src/ram.rs) over
// an engine's retained tree, with the per-client "already forwarded" marks kept, checked and set on the device.
//
//   k_ms_mark      inserts mark words into the mark set (store-time marks)
//   k_ms_rebuild   re-inserts the mark set into a larger table, dropping the entries of retired handles
//   k_ms_filter    one thread per matched handle of a lookup: drops what was already forwarded to the query, counts the rest
//                  per query, or lists it as a candidate when the query shares a key with another query of the batch
//   k_ms_claim_init, k_ms_claim, k_ms_decide   the rounds that deliver contested candidates in batch order
//   k_ms_scan      per-query survivor counts -> spans
//   k_ms_deliver   compacts the survivors into the output and marks them as forwarded
//
// The mark set is an open-addressing table of u64 words  handle << 32 | kind << 31 | key  (kind 0: client key, 1: share key;
// ~0 = empty), filled by 64-bit CAS and kept at load <= 1/2.  The device is its only owner.
//
// MsCore<Backend> is the store's host logic, written once for the product (msgstore.cu: CUDA runtime and the engine's ABI) and
// the CPU emulation (tests/native/emu/emu_msgstore.cpp: host memory and the emulated retained lookup).  A Backend provides
//   Buf                      device memory: .p, ensure(bytes) -> gm status (contents are not kept when it grows)
//   h2d / d2h / fill / sync  copies, a byte fill and a wait on the store's stream -> gm status
//   stream()                 the stream every launch goes to
//   device()                 false on a host-only engine: lookups return GM_ERR_NO_DEVICE
//   walk(...)                gm_retain_match_batch_device_at into device buffers
//   set_ttl / bulk_ttl / remove_batch / remove_expired   the engine's gm_retain_set_ttl, gm_retain_bulk_load_ttl,
//                            gm_retain_remove_batch, gm_retain_remove_expired
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/gpumqtt.h"
#include "layout.h"

#ifndef GM_LAUNCH
#ifdef GM_CPU_EMU
#define GM_LAUNCH(k, grid, block, smem, s, ...) emu::launch(dim3(grid), dim3(block), [&] { k(__VA_ARGS__); })
#else
#define GM_LAUNCH(k, grid, block, smem, s, ...) k<<<grid, block, smem, s>>>(__VA_ARGS__)
#endif
#endif

#ifndef GM_TRY
#define GM_TRY(expr) do { const int32_t _st = (expr); if (_st != GM_OK) return _st; } while (0)
#endif

namespace gm {

extern thread_local std::string g_err;   // the text of gm_last_error

constexpr u64 MS_EMPTY = ~0ull;
constexpr u32 MS_NONE = 0xFFFFFFFFu;
constexpr u32 MS_KEY_LIMIT = 1u << 31;

GM_HD u64 ms_word(u32 handle, u32 kind, u32 key) { return static_cast<u64>(handle) << 32 | static_cast<u64>(kind) << 31 | key; }

GM_HD u64 ms_hash(u64 x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull;
    return x ^ (x >> 33);
}

__device__ __forceinline__ bool ms_contains(const u64* __restrict__ t, u64 mask, u64 w) {
    for (u64 i = ms_hash(w) & mask;; i = (i + 1) & mask) {
        const u64 v = t[i];
        if (v == w) return true;
        if (v == MS_EMPTY) return false;
    }
}

// inserts w unless present; returns its slot.  The table always has an empty slot (load <= 1/2).
__device__ __forceinline__ u64 ms_insert(u64* t, u64 mask, u64 w, unsigned long long* count) {
    for (u64 i = ms_hash(w) & mask;; i = (i + 1) & mask) {
        u64 v = t[i];
        if (v == MS_EMPTY) {
            v = atomicCAS(reinterpret_cast<unsigned long long*>(t + i), MS_EMPTY, w);
            if (v == MS_EMPTY) { if (count) atomicAdd(count, 1ull); return i; }
        }
        if (v == w) return i;
    }
}

struct MsCtl {                      // per-call counters (zeroed before the lookup's kernels)
    unsigned long long ncand;       // contested candidates listed by k_ms_filter
    unsigned long long undecided;   // candidates left undecided by the last round
    unsigned long long total;       // handles delivered by the call (k_ms_scan)
};

struct MsGet {                      // one lookup's buffers (all device)
    const uint2* raw_spans; const u32* raw; u64 raw_total; u32 n;
    const u32* clients; const u32* shares; const u8* contested;
    const u64* marks; u64 mask;     // the mark set
    u32* owner; u8* keep;           // [raw_total]: query of each matched handle; 0 drop, 1 deliver, 2 contested (until decided)
    u32* cnt; u32* base; u32* cur;  // [n]
    u32* cand; u8* state;           // [raw_total]: contested candidates (raw index), 0 undecided, 1 delivered, 2 rejected
    u64* ckeys; u64* cclaim; u8* ctaken; u32* cslot; u64 cmask;   // the per-call claim table and each candidate's two slots
    uint2* spans; u32* out;
    MsCtl* ctl;
};

__global__ void __launch_bounds__(256) k_ms_mark(u64* t, u64 mask, const u64* __restrict__ words, u64 n, unsigned long long* count) {
    for (u64 i = blockIdx.x * static_cast<u64>(blockDim.x) + threadIdx.x; i < n; i += static_cast<u64>(gridDim.x) * blockDim.x)
        ms_insert(t, mask, words[i], count);
}

__global__ void __launch_bounds__(256) k_ms_rebuild(const u64* __restrict__ old, u64 n_old, u64* t, u64 mask, const u32* __restrict__ retired, u64 n_retired_bits,
                                                    unsigned long long* count) {
    for (u64 i = blockIdx.x * static_cast<u64>(blockDim.x) + threadIdx.x; i < n_old; i += static_cast<u64>(gridDim.x) * blockDim.x) {
        const u64 w = old[i];
        if (w == MS_EMPTY) continue;
        const u32 h = static_cast<u32>(w >> 32);
        if (h < n_retired_bits && (retired[h >> 5] >> (h & 31) & 1u)) continue;
        ms_insert(t, mask, w, count);
    }
}

// the query a matched handle belongs to: the retained lookup's spans are an exclusive scan of its per-query counts
__device__ __forceinline__ u32 ms_owner(const uint2* __restrict__ spans, u32 n, u64 j) {
    u32 lo = 0, hi = n;              // first query whose span starts after j, minus one
    while (lo < hi) { const u32 mid = (lo + hi) >> 1; if (spans[mid].x <= j) lo = mid + 1; else hi = mid; }
    return lo - 1;
}

__global__ void __launch_bounds__(256) k_ms_filter(MsGet p) {
    for (u64 j = blockIdx.x * static_cast<u64>(blockDim.x) + threadIdx.x; j < p.raw_total; j += static_cast<u64>(gridDim.x) * blockDim.x) {
        const u32 q = ms_owner(p.raw_spans, p.n, j);
        const u32 h = p.raw[j], c = p.clients[q], s = p.shares[q];
        p.owner[j] = q;
        bool fwd = ms_contains(p.marks, p.mask, ms_word(h, 0, c));
        if (!fwd && s != MS_NONE) fwd = ms_contains(p.marks, p.mask, ms_word(h, 1, s));
        u8 k = 0;
        if (!fwd) {
            if (p.contested[q]) {
                k = 2;
                p.cand[atomicAdd(&p.ctl->ncand, 1ull)] = static_cast<u32>(j);
            } else {
                k = 1;
                atomicAdd(p.cnt + q, 1u);
            }
        }
        p.keep[j] = k;
    }
}

// the claim table holds the keys of the contested candidates; cslot[2k + i] = slot of candidate k's key i (MS_NONE: no share key)
__global__ void __launch_bounds__(256) k_ms_claim_init(MsGet p, u64 ncand) {
    for (u64 k = blockIdx.x * static_cast<u64>(blockDim.x) + threadIdx.x; k < ncand; k += static_cast<u64>(gridDim.x) * blockDim.x) {
        const u32 j = p.cand[k], q = p.owner[j], h = p.raw[j], s = p.shares[q];
        p.state[k] = 0;
        p.cslot[2 * k] = static_cast<u32>(ms_insert(p.ckeys, p.cmask, ms_word(h, 0, p.clients[q]), nullptr));
        p.cslot[2 * k + 1] = s == MS_NONE ? MS_NONE : static_cast<u32>(ms_insert(p.ckeys, p.cmask, ms_word(h, 1, s), nullptr));
    }
}

// One round, step 1: an undecided candidate whose key a delivered candidate took is rejected; the others claim each of their
// keys for this round.  A claim is round << 32 | ~raw index: atomicMax keeps the smallest raw index (batch order) of the round.
__global__ void __launch_bounds__(256) k_ms_claim(MsGet p, u64 ncand, u32 round) {
    for (u64 k = blockIdx.x * static_cast<u64>(blockDim.x) + threadIdx.x; k < ncand; k += static_cast<u64>(gridDim.x) * blockDim.x) {
        if (p.state[k]) continue;
        const u32 s0 = p.cslot[2 * k], s1 = p.cslot[2 * k + 1];
        if (p.ctaken[s0] || (s1 != MS_NONE && p.ctaken[s1])) { p.state[k] = 2; continue; }
        const u64 mine = static_cast<u64>(round) << 32 | static_cast<u32>(~p.cand[k]);
        atomicMax(reinterpret_cast<unsigned long long*>(p.cclaim + s0), mine);
        if (s1 != MS_NONE) atomicMax(reinterpret_cast<unsigned long long*>(p.cclaim + s1), mine);
    }
}

// step 2: a candidate that holds the claim of every key it has is delivered and takes them (two such candidates share no key)
__global__ void __launch_bounds__(256) k_ms_decide(MsGet p, u64 ncand, u32 round) {
    for (u64 k = blockIdx.x * static_cast<u64>(blockDim.x) + threadIdx.x; k < ncand; k += static_cast<u64>(gridDim.x) * blockDim.x) {
        if (p.state[k]) continue;
        const u32 j = p.cand[k], s0 = p.cslot[2 * k], s1 = p.cslot[2 * k + 1];
        const u64 mine = static_cast<u64>(round) << 32 | static_cast<u32>(~j);
        if (p.cclaim[s0] == mine && (s1 == MS_NONE || p.cclaim[s1] == mine)) {
            p.state[k] = 1;
            p.ctaken[s0] = 1;
            if (s1 != MS_NONE) p.ctaken[s1] = 1;
            p.keep[j] = 1;
            atomicAdd(p.cnt + p.owner[j], 1u);
        } else {
            atomicAdd(&p.ctl->undecided, 1ull);
        }
    }
}

__global__ void __launch_bounds__(1024) k_ms_scan(MsGet p) {
    __shared__ unsigned long long s_part[1024];
    const u32 tid = threadIdx.x, nq = p.n;
    const u32 per = (nq + 1023) / 1024;
    const u32 b = min(nq, tid * per), e = min(nq, b + per);
    unsigned long long sum = 0;
    for (u32 i = b; i < e; ++i) sum += p.cnt[i];
    s_part[tid] = sum;
    __syncthreads();
    if (tid == 0) {
        unsigned long long run = 0;
        for (int i = 0; i < 1024; ++i) { const unsigned long long x = s_part[i]; s_part[i] = run; run += x; }
        p.ctl->total = run;
    }
    __syncthreads();
    unsigned long long run = s_part[tid];
    for (u32 i = b; i < e; ++i) {
        const u32 c = p.cnt[i];
        const u32 off = run > 0xFFFFFFFFull ? 0xFFFFFFFFu : static_cast<u32>(run);
        p.base[i] = off;
        p.spans[i] = make_uint2(off, c);
        run += c;
    }
}

// only when the output holds every delivered handle: write it and mark it as forwarded to its query
__global__ void __launch_bounds__(256) k_ms_deliver(MsGet p, u64* marks, unsigned long long* count) {
    for (u64 j = blockIdx.x * static_cast<u64>(blockDim.x) + threadIdx.x; j < p.raw_total; j += static_cast<u64>(gridDim.x) * blockDim.x) {
        if (p.keep[j] != 1) continue;
        const u32 q = p.owner[j], h = p.raw[j], s = p.shares[q];
        p.out[p.base[q] + atomicAdd(p.cur + q, 1u)] = h;
        ms_insert(marks, p.mask, ms_word(h, 0, p.clients[q]), count);
        if (s != MS_NONE) ms_insert(marks, p.mask, ms_word(h, 1, s), count);
    }
}

inline unsigned ms_grid(u64 n, int num_sms) { return static_cast<unsigned>(std::max<u64>(1, std::min<u64>((n + 255) / 256, static_cast<u64>(num_sms) * 8))); }

// ================================================================================================================================
template <class B>
struct MsCore {
    using Buf = typename B::Buf;
    B be;
    std::mutex mu;
    int num_sms = 132;
    // host bookkeeping, one bit per handle
    std::vector<u32> live, retired;
    u64 messages = 0, n_retired = 0;
    bool purge_needed = false;      // a retired handle was stored again: its old marks must go before the next lookup
    std::vector<u64> pending;       // store-time marks not yet inserted (k_ms_mark before the next lookup)
    // the mark set
    Buf tbl[2], d_count, d_pending, d_retired;
    int act = 0;                    // tbl[act] is the mark set; a rebuild fills the other one
    u64 slots = 0, marks = 0;       // marks: live entries as of the last device read, plus pending ones inserted since (a bound)
    u64 init_slots = 1u << 16, rehashes = 0, purges = 0;
    // lookup scratch
    Buf d_blob, d_offs, d_clients, d_shares, d_contested, d_rspans, d_status, d_raw, d_owner, d_keep, d_cnt, d_base, d_cur, d_cand, d_state, d_ckeys, d_cclaim,
        d_ctaken, d_cslot, d_spans, d_out, d_ctl;
    u64 raw_cap = 1u << 16;
    std::vector<char> h_blob;
    std::vector<u32> h_offs;
    std::vector<u8> h_contested;

    template <class... A> explicit MsCore(A&&... a) : be(std::forward<A>(a)...) {}

    static bool bit(const std::vector<u32>& v, u32 h) { return (h >> 5) < v.size() && (v[h >> 5] >> (h & 31) & 1u); }
    static void set_bit(std::vector<u32>& v, u32 h, bool on) {
        if ((h >> 5) >= v.size()) { if (!on) return; v.resize((h >> 5) + 1, 0); }
        if (on) v[h >> 5] |= 1u << (h & 31); else v[h >> 5] &= ~(1u << (h & 31));
    }

    // ---- store ----------------------------------------------------------------------------------------------------------
    static int check_marks(const u32* clients, const u32* shares, u32 n) {
        for (u32 i = 0; i < n; ++i)
            if (clients[i] >= MS_KEY_LIMIT || (shares && shares[i] != MS_NONE && shares[i] >= MS_KEY_LIMIT)) {
                g_err = "client and share keys are below 2^31"; return GM_ERR_INVALID_ARG;
            }
        return GM_OK;
    }
    int check_message(u32 handle, u64 expiry) const {
        if (handle >= GM_RETAIN_TTL_MAX_HANDLE) { g_err = "message handles are below GM_RETAIN_TTL_MAX_HANDLE"; return GM_ERR_INVALID_ARG; }
        if (expiry >= ~0ull) { g_err = "expiry_time_at must be below UINT64_MAX"; return GM_ERR_INVALID_ARG; }
        if (bit(live, handle)) { g_err = "the handle is stored already: a handle is stored again only after the sweep removed it"; return GM_ERR_INVALID_ARG; }
        return GM_OK;
    }
    static void append_key(std::string& k, const char* topic, u32 len, u32 handle) {   // topic.push(Level::Normal(msg_id.to_string()))
        k.append(topic, len);
        k.push_back('/');
        k += std::to_string(handle);
    }
    // BTreeMap::insert per (client, share): the last entry for a client wins
    void queue_marks(u32 handle, const u32* clients, const u32* shares, u32 n) {
        std::unordered_map<u32, u32> seen;
        for (u32 i = n; i-- > 0;) {
            if (!seen.emplace(clients[i], 0).second) continue;
            pending.push_back(ms_word(handle, 0, clients[i]));
            if (shares && shares[i] != MS_NONE) pending.push_back(ms_word(handle, 1, shares[i]));
        }
    }
    void stored(u32 handle) {
        set_bit(live, handle, true);
        messages++;
        if (bit(retired, handle)) purge_needed = true;
    }

    int store(const char* topic, u32 len, u32 handle, u64 expiry, const u32* clients, const u32* shares, u32 n_marks) {
        if ((!topic && len) || (n_marks && !clients)) return GM_ERR_INVALID_ARG;
        std::lock_guard<std::mutex> g(mu);
        GM_TRY(check_message(handle, expiry));
        GM_TRY(check_marks(clients, shares, n_marks));
        std::string key;
        append_key(key, topic, len, handle);
        GM_TRY(be.set_ttl(key.data(), static_cast<u32>(key.size()), handle, expiry + 1));
        stored(handle);
        queue_marks(handle, clients, shares, n_marks);
        return GM_OK;
    }

    int store_batch(const char* blob, const uint32_t* offsets, const uint32_t* handles, const uint64_t* expiry, uint64_t n, const uint32_t* mark_offsets,
                    const uint32_t* clients, const uint32_t* shares) {
        if (n && (!blob || !offsets || !handles || !expiry)) return GM_ERR_INVALID_ARG;
        if (mark_offsets && n && mark_offsets[n] && !clients) return GM_ERR_INVALID_ARG;
        std::lock_guard<std::mutex> g(mu);
        std::vector<u32> batch;
        for (u64 i = 0; i < n; ++i) {
            GM_TRY(check_message(handles[i], expiry[i]));
            if (bit(batch, handles[i])) { g_err = "a handle appears twice in the batch"; return GM_ERR_INVALID_ARG; }
            set_bit(batch, handles[i], true);
            if (mark_offsets) {
                if (mark_offsets[i + 1] < mark_offsets[i]) return GM_ERR_INVALID_ARG;
                GM_TRY(check_marks(clients + mark_offsets[i], shares ? shares + mark_offsets[i] : nullptr, mark_offsets[i + 1] - mark_offsets[i]));
            }
        }
        std::string keys;
        std::vector<u32> koffs(n + 1, 0);
        std::vector<u64> dl(n);
        for (u64 i = 0; i < n; ++i) {
            append_key(keys, blob + offsets[i], offsets[i + 1] - offsets[i], handles[i]);
            if (keys.size() > 0xFFFFFFFFull) { g_err = "key blob >= 4 GiB"; return GM_ERR_TOO_LARGE; }
            koffs[i + 1] = static_cast<u32>(keys.size());
            dl[i] = expiry[i] + 1;
        }
        u64 n_set = 0;
        GM_TRY(be.bulk_ttl(keys.data(), koffs.data(), handles, dl.data(), n, &n_set));
        if (n_set != n) {               // an invalid topic: take the valid ones out again
            GM_TRY(be.remove_batch(keys.data(), koffs.data(), n));
            g_err = "invalid topic in the batch";
            return GM_ERR_INVALID_TOPIC;
        }
        for (u64 i = 0; i < n; ++i) {
            stored(handles[i]);
            if (mark_offsets)
                queue_marks(handles[i], clients + mark_offsets[i], shares ? shares + mark_offsets[i] : nullptr, mark_offsets[i + 1] - mark_offsets[i]);
        }
        return GM_OK;
    }

    // ---- sweep: remove_expired_messages (ram.rs:143-191) removes when expiry_time_at <= now -------------------------------
    int remove_expired(u64 now, u32* out, u64 cap, u64* n_removed) {
        if (cap && !out) return GM_ERR_INVALID_ARG;
        std::lock_guard<std::mutex> g(mu);
        u64 n = 0;
        GM_TRY(be.remove_expired(now == ~0ull ? now : now + 1, out, cap, &n));
        for (u64 i = 0; i < n; ++i) {
            set_bit(live, out[i], false);
            if (!bit(retired, out[i])) { set_bit(retired, out[i], true); n_retired++; }
            messages--;
        }
        if (n && !pending.empty())      // store-time marks of a removed handle die with it
            pending.erase(std::remove_if(pending.begin(), pending.end(), [&](u64 w) { return !bit(live, static_cast<u32>(w >> 32)); }), pending.end());
        if (n_removed) *n_removed = n;
        return GM_OK;
    }

    // ---- the mark set ---------------------------------------------------------------------------------------------------
    int read_count() {
        unsigned long long c = 0;
        GM_TRY(be.d2h(&c, d_count.p, sizeof(c)));
        GM_TRY(be.sync());
        marks = c;
        return GM_OK;
    }
    int init_device() {
        if (slots) return GM_OK;
        GM_TRY(d_count.ensure(sizeof(unsigned long long)));
        GM_TRY(be.fill(d_count.p, 0, sizeof(unsigned long long)));
        GM_TRY(tbl[act].ensure(init_slots * sizeof(u64)));
        GM_TRY(be.fill(tbl[act].p, 0xFF, init_slots * sizeof(u64)));
        slots = init_slots;
        marks = 0;
        return GM_OK;
    }
    // re-insert into a table that holds `need` entries at load <= 1/2, dropping the entries of retired handles
    int rebuild(u64 need) {
        u64 ns = slots;
        while (ns < 2 * need) ns *= 2;
        Buf& nt = tbl[act ^ 1];
        GM_TRY(nt.ensure(ns * sizeof(u64)));
        GM_TRY(be.fill(nt.p, 0xFF, ns * sizeof(u64)));
        GM_TRY(be.fill(d_count.p, 0, sizeof(unsigned long long)));
        const u64 nbits = static_cast<u64>(retired.size()) * 32;
        if (!retired.empty()) {
            GM_TRY(d_retired.ensure(retired.size() * sizeof(u32)));
            GM_TRY(be.h2d(d_retired.p, retired.data(), retired.size() * sizeof(u32)));
        }
        GM_LAUNCH(k_ms_rebuild, ms_grid(slots, num_sms), 256, 0, be.stream(), static_cast<const u64*>(tbl[act].p), slots, static_cast<u64*>(nt.p), ns - 1,
                  static_cast<const u32*>(d_retired.p), retired.empty() ? 0 : nbits, static_cast<unsigned long long*>(d_count.p));
        GM_TRY(be.launched());
        act ^= 1;
        if (ns != slots) rehashes++;
        if (n_retired) purges++;
        slots = ns;
        retired.clear();
        n_retired = 0;
        purge_needed = false;
        return read_count();
    }
    int ensure_room(u64 extra) {
        if (purge_needed || 2 * (marks + extra) > slots) return rebuild(marks + extra);
        return GM_OK;
    }
    int flush_pending() {
        GM_TRY(init_device());
        GM_TRY(ensure_room(pending.size()));
        if (pending.empty()) return GM_OK;
        GM_TRY(d_pending.ensure(pending.size() * sizeof(u64)));
        GM_TRY(be.h2d(d_pending.p, pending.data(), pending.size() * sizeof(u64)));
        GM_LAUNCH(k_ms_mark, ms_grid(pending.size(), num_sms), 256, 0, be.stream(), static_cast<u64*>(tbl[act].p), slots - 1, static_cast<const u64*>(d_pending.p),
                  static_cast<u64>(pending.size()), static_cast<unsigned long long*>(d_count.p));
        GM_TRY(be.launched());
        marks += pending.size();
        GM_TRY(be.sync());              // (d_pending is reused by the next flush)
        pending.clear();
        return GM_OK;
    }

    // ---- get (ram.rs:303-367) for a batch, in batch order ---------------------------------------------------------------
    int get_batch(u64 now, const char* blob, const uint32_t* offsets, uint64_t n, const uint32_t* clients, const uint32_t* shares, gm_span* out_spans,
                  uint32_t* out_handles, uint64_t cap, uint64_t* needed, int32_t* status) {
        if ((n && (!offsets || !out_spans || !status || !clients || !shares)) || (cap && !out_handles)) return GM_ERR_INVALID_ARG;
        if (needed) *needed = 0;
        if (n == 0) return GM_OK;
        if (n > 0xFFFFFFF0ull) { g_err = "filter batch too large"; return GM_ERR_TOO_LARGE; }
        GM_TRY(check_marks(clients, shares, static_cast<u32>(n)));
        if (!be.device()) { g_err = "host-only engine cannot match: there is no CPU fallback"; return GM_ERR_NO_DEVICE; }
        std::lock_guard<std::mutex> g(mu);
        // the filters with the level get appends: '+' unless the last level is '#'
        h_blob.clear(); h_offs.assign(n + 1, 0);
        for (u64 i = 0; i < n; ++i) {
            const char* f = blob + offsets[i];
            const u32 len = offsets[i + 1] - offsets[i];
            h_blob.insert(h_blob.end(), f, f + len);
            const bool hash_last = len && f[len - 1] == '#' && (len == 1 || f[len - 2] == '/');
            if (!hash_last) { h_blob.push_back('/'); h_blob.push_back('+'); }
            if (h_blob.size() > 0xFFFFFFF0ull) { g_err = "filter blob >= 4 GiB"; return GM_ERR_TOO_LARGE; }
            h_offs[i + 1] = static_cast<u32>(h_blob.size());
        }
        // queries that share a client key or a share key with another query of the batch
        std::unordered_map<u64, u32> uses;
        uses.reserve(2 * n);
        for (u64 i = 0; i < n; ++i) { uses[clients[i]]++; if (shares[i] != MS_NONE) uses[1ull << 32 | shares[i]]++; }
        h_contested.assign(n, 0);
        bool any_contested = false;
        for (u64 i = 0; i < n; ++i) {
            h_contested[i] = uses[clients[i]] > 1 || (shares[i] != MS_NONE && uses[1ull << 32 | shares[i]] > 1);
            any_contested |= h_contested[i] != 0;
        }
        const u64 bytes = h_blob.size();
        GM_TRY(d_blob.ensure(bytes + 16));
        GM_TRY(d_offs.ensure((n + 1) * sizeof(u32)));
        GM_TRY(d_clients.ensure(n * sizeof(u32)));
        GM_TRY(d_shares.ensure(n * sizeof(u32)));
        GM_TRY(d_contested.ensure(n));
        GM_TRY(d_rspans.ensure(n * sizeof(gm_span)));
        GM_TRY(d_status.ensure(n * sizeof(int32_t)));
        GM_TRY(d_cnt.ensure(n * sizeof(u32)));
        GM_TRY(d_base.ensure(n * sizeof(u32)));
        GM_TRY(d_cur.ensure(n * sizeof(u32)));
        GM_TRY(d_spans.ensure(n * sizeof(gm_span)));
        GM_TRY(d_ctl.ensure(sizeof(MsCtl)));
        if (bytes) GM_TRY(be.h2d(d_blob.p, h_blob.data(), bytes));
        GM_TRY(be.h2d(d_offs.p, h_offs.data(), (n + 1) * sizeof(u32)));
        GM_TRY(be.h2d(d_clients.p, clients, n * sizeof(u32)));
        GM_TRY(be.h2d(d_shares.p, shares, n * sizeof(u32)));
        GM_TRY(be.h2d(d_contested.p, h_contested.data(), n));
        GM_TRY(flush_pending());
        // the tree: every live matched handle, per query
        u64 raw_total = 0;
        for (;;) {
            GM_TRY(d_raw.ensure(raw_cap * sizeof(u32)));
            const int st = be.walk(now, d_blob.p, bytes, static_cast<const u32*>(d_offs.p), n, static_cast<gm_span*>(d_rspans.p), static_cast<u32*>(d_raw.p), raw_cap,
                                   &raw_total, static_cast<int32_t*>(d_status.p));
            if (st == GM_OK) break;
            if (st != GM_ERR_CAPACITY) return st;
            raw_cap = std::max(raw_total, 2 * raw_cap);
        }
        // room for what this call can mark: two entries per delivered handle, at most cap of them
        GM_TRY(ensure_room(2 * std::min<u64>(cap, raw_total)));
        const u64 rt = std::max<u64>(raw_total, 1);
        GM_TRY(d_owner.ensure(rt * sizeof(u32)));
        GM_TRY(d_keep.ensure(rt));
        GM_TRY(d_cand.ensure(rt * sizeof(u32)));
        MsGet p{};
        p.raw_spans = static_cast<const uint2*>(d_rspans.p); p.raw = static_cast<const u32*>(d_raw.p); p.raw_total = raw_total; p.n = static_cast<u32>(n);
        p.clients = static_cast<const u32*>(d_clients.p); p.shares = static_cast<const u32*>(d_shares.p);
        p.contested = static_cast<const u8*>(d_contested.p);
        p.marks = static_cast<const u64*>(tbl[act].p); p.mask = slots - 1;
        p.owner = static_cast<u32*>(d_owner.p); p.keep = static_cast<u8*>(d_keep.p);
        p.cnt = static_cast<u32*>(d_cnt.p); p.base = static_cast<u32*>(d_base.p); p.cur = static_cast<u32*>(d_cur.p);
        p.cand = static_cast<u32*>(d_cand.p);
        p.spans = static_cast<uint2*>(d_spans.p); p.out = nullptr;
        p.ctl = static_cast<MsCtl*>(d_ctl.p);
        GM_TRY(be.fill(d_ctl.p, 0, sizeof(MsCtl)));
        GM_TRY(be.fill(d_cnt.p, 0, n * sizeof(u32)));
        if (raw_total) {
            GM_LAUNCH(k_ms_filter, ms_grid(raw_total, num_sms), 256, 0, be.stream(), p);
            GM_TRY(be.launched());
        }
        if (any_contested && raw_total) GM_TRY(resolve(p));
        GM_LAUNCH(k_ms_scan, 1, 1024, 0, be.stream(), p);
        GM_TRY(be.launched());
        MsCtl h{};
        GM_TRY(be.d2h(&h, d_ctl.p, sizeof(MsCtl)));
        GM_TRY(be.d2h(status, d_status.p, n * sizeof(int32_t)));
        GM_TRY(be.d2h(out_spans, d_spans.p, n * sizeof(gm_span)));
        GM_TRY(be.sync());
        if (needed) *needed = h.total;
        if (h.total > 0xFFFFFFFFull) { g_err = "batch produces >= 2^32 handles: split it"; return GM_ERR_TOO_LARGE; }
        if (h.total > cap) { g_err = "out_handles too small"; return GM_ERR_CAPACITY; }
        if (!h.total) return GM_OK;
        GM_TRY(d_out.ensure(h.total * sizeof(u32)));
        p.out = static_cast<u32*>(d_out.p);
        GM_TRY(be.fill(d_cur.p, 0, n * sizeof(u32)));
        GM_LAUNCH(k_ms_deliver, ms_grid(raw_total, num_sms), 256, 0, be.stream(), p, static_cast<u64*>(tbl[act].p), static_cast<unsigned long long*>(d_count.p));
        GM_TRY(be.launched());
        GM_TRY(be.d2h(out_handles, d_out.p, h.total * sizeof(u32)));
        return read_count();            // (synchronises)
    }

    // rounds over the contested candidates until every one is delivered or rejected (each round decides at least the first)
    int resolve(MsGet& p) {
        MsCtl h{};
        GM_TRY(be.d2h(&h, d_ctl.p, sizeof(MsCtl)));
        GM_TRY(be.sync());
        const u64 nc = h.ncand;
        if (!nc) return GM_OK;
        u64 cs = 64;
        while (cs < 4 * nc) cs *= 2;
        GM_TRY(d_state.ensure(nc));
        GM_TRY(d_cslot.ensure(2 * nc * sizeof(u32)));
        GM_TRY(d_ckeys.ensure(cs * sizeof(u64)));
        GM_TRY(d_cclaim.ensure(cs * sizeof(u64)));
        GM_TRY(d_ctaken.ensure(cs));
        GM_TRY(be.fill(d_ckeys.p, 0xFF, cs * sizeof(u64)));
        GM_TRY(be.fill(d_cclaim.p, 0, cs * sizeof(u64)));
        GM_TRY(be.fill(d_ctaken.p, 0, cs));
        p.state = static_cast<u8*>(d_state.p); p.cslot = static_cast<u32*>(d_cslot.p);
        p.ckeys = static_cast<u64*>(d_ckeys.p); p.cclaim = static_cast<u64*>(d_cclaim.p); p.ctaken = static_cast<u8*>(d_ctaken.p); p.cmask = cs - 1;
        const unsigned grid = ms_grid(nc, num_sms);
        GM_LAUNCH(k_ms_claim_init, grid, 256, 0, be.stream(), p, nc);
        GM_TRY(be.launched());
        for (u32 round = 1;; ++round) {
            GM_TRY(be.fill(&p.ctl->undecided, 0, sizeof(unsigned long long)));
            GM_LAUNCH(k_ms_claim, grid, 256, 0, be.stream(), p, nc, round);
            GM_LAUNCH(k_ms_decide, grid, 256, 0, be.stream(), p, nc, round);
            GM_TRY(be.launched());
            GM_TRY(be.d2h(&h, d_ctl.p, sizeof(MsCtl)));
            GM_TRY(be.sync());
            if (!h.undecided) return GM_OK;
        }
    }

    int stats(gm_msgstore_stats* out) {
        std::lock_guard<std::mutex> g(mu);
        if (slots) GM_TRY(read_count());
        out->messages = messages;
        out->marks = slots ? marks : 0;
        out->pending_marks = pending.size();
        out->mark_slots = slots;
        out->rehashes = rehashes;
        out->purges = purges;
        out->retired = n_retired;
        return GM_OK;
    }
};

}  // namespace gm
