// sm_90a kernels of the SUBSCRIBE -> retained-message lookup (RetainTree::matches,
// rmqtt/src/retain.rs:291-367) for a batch of topic filters.
//
// A query is a FILTER, so its work is data dependent: an exact filter touches one path, `reg/+/+/...`
// fans out to tens of thousands of nodes.  The batch is walked in ROUNDS of wildcard expansions: round 0 follows
// every filter's literal prefix from the root (one thread per query); a '+' (or a '#' that cannot use the range
// shortcut) becomes TASKS — chunks of the node's contiguous child block — that the next round's warps read
// coalesced, one child per lane, each lane then following the filter's exact levels below its child in place.
// '#' is normally a single contiguous range of the pre-order value array (retain_tree.h).  Matched values are
// recorded as descriptors and expanded into per-query contiguous lists by k_retain_expand.
#pragma once
#include <cuda_runtime.h>

#include "kernels.cuh"
#include "retain_tree.h"

namespace gm {

struct alignas(16) RDesc { u32 q, ref, cnt, kind; };   // kind 0: the value itself, 1: rvals[ref .. ref+cnt)

// A TASK = "expand the child block [kb, kb+kn) of one node for query q whose filter is at position pos":
//   mode 1  the filter level at pos is '+'   (retain.rs:324-342): every child continues at pos+1
//   mode 2  the filter level at pos is '#' and a literal "#" child hides somewhere below (retain.rs:343-365): every child
//           is emitted and continues at the SAME pos, one tree level per round
// Tasks exist only at WILDCARD levels.  Everything between two wildcards — the chain of exact (literal) levels — is
// followed inside the thread that holds the node (one hash probe per level, nothing written): round-1's kernel moved
// every visited node through a global queue (32 B written + 32 B re-read per visit) and needed one launch per tree level.
struct alignas(16) RTask { u32 q, pos_mode, kb, kn; };   // pos_mode = pos | mode << 30
constexpr u32 RTASK_CHUNK = 256;                         // child-block entries per task: large blocks are split so that warps balance

// Work queues (tasks, descriptor list) are split into RQ slices with one counter each: a single bump counter serialises
// the appends of a C4 batch on one L2 atomic unit.
constexpr u32 RQ = 64;

struct RetainParams {
    RetainView v;
    const u32* qtok8;    // [nq][8]  filter levels 0..7
    const u32* qtok;     // [tok_levels][nq]  levels >= 8
    const u32* qmeta;    // [nq]
    u32 nq, tok_levels;  // nq: rows of the launch (the row stride of qtok); with n_ptr a capacity
    const u32* n_ptr;    // small-batch graphs: the real filter count lives in device memory (rows at or past it are not touched)
    RDesc* descs;
    u32* n_desc;         // [RQ]
    u32 cap_items, cap_desc;   // per SLICE
    u32* qtotal;         // [nq] matched values per query
    u32* err;            // bit 0: task-queue overflow, bit 1: descriptor overflow
    unsigned long long* stats;   // optional [2]: nodes visited, hash probes issued (diagnostics)
    // Deadlines (read by the TTL instantiations only; kept last so that the other instantiations see an unchanged layout):
    // dl[handle] in ms since the Unix epoch, ~0 = none; handles at or past n_dl never expire.  `now` lives in device memory,
    // so a captured graph reads the current one at every launch.
    const u64* dl;
    u32 n_dl;
    const u64* now;
};

// a handle is live at `now` unless its deadline has come (TimedValue::is_expired: now >= deadline)
__device__ __forceinline__ bool retain_live(const u64* dl, u32 n_dl, u64 now, u32 v) { return v >= n_dl || now < dl[v]; }

__device__ __forceinline__ u32 retain_tok(const RetainParams& p, u32 q, u32 pos) {
    return pos < TOK8 ? p.qtok8[static_cast<size_t>(q) * TOK8 + pos] : p.qtok[static_cast<size_t>(pos) * p.nq + q];
}

// exact child lookup: the slot carries the child's whole record
__device__ __forceinline__ bool retain_child(const RetainView& v, u32 node, u32 token, u32 (&s)[8]) {
    u32 idx = redge_hash(node, token) & v.edge_mask;
    for (;;) {
        ld256(v.edges + idx, s);
        if (s[2] == 0) return false;
        if (s[0] == node && s[1] == token) return true;
        idx = (idx + 1) & v.edge_mask;
    }
}

// block-wide: exclusive prefix of the (clamped) slice counts into s_pre[RQ + 1]; returns the total
__device__ __forceinline__ u32 queue_prefix(const u32* __restrict__ counters, u32 slice_cap, u32* s_pre) {
    if (threadIdx.x == 0) {
        u32 run = 0;
        for (u32 k = 0; k < RQ; ++k) { s_pre[k] = run; run += min(counters[k], slice_cap); }
        s_pre[RQ] = run;
    }
    __syncthreads();
    return s_pre[RQ];
}
// logical index g -> physical index inside the sliced array
__device__ __forceinline__ size_t queue_locate(const u32* s_pre, u32 g, u32 slice_cap) {
    u32 lo = 0;
#pragma unroll
    for (u32 step = RQ / 2; step; step >>= 1) if (s_pre[lo + step] <= g) lo += step;
    return static_cast<size_t>(lo) * slice_cap + (g - s_pre[lo]);
}

// per-lane appends (called from divergent code): one atomic on the lane's slice counter
__device__ __forceinline__ void emit_desc(const RetainParams& p, u32 sq, u32 q, u32 ref, u32 cnt, u32 kind) {
    atomicAdd(p.qtotal + q, cnt);
    const u32 at = atomicAdd(p.n_desc + sq, 1u);
    if (at < p.cap_desc) p.descs[static_cast<size_t>(sq) * p.cap_desc + at] = RDesc{q, ref, cnt, kind}; else atomicOr(p.err, 2u);
}
// one matched value: with deadlines, an expired one is neither counted nor recorded
template <bool TTL>
__device__ __forceinline__ void emit_value(const RetainParams& p, u64 now, u32 sq, u32 q, u32 v) {
    if (!TTL || retain_live(p.dl, p.n_dl, now, v)) emit_desc(p, sq, q, v, 1u, 0u);
}
// LOCALITY: a task goes into the queue slice of its child block's POSITION IN THE TREE (child blocks are laid out in tree
// pre-order), not of the warp that produced it.  The next round consumes the slices one after another, so all the tasks
// that expand the same part of the tree — dozens of filters such as `+/+/+/…` and `reg/+/+/…` cover every site block — run
// close together in time and share the child blocks and the hash slots of the nodes below through L2, instead of each
// filter streaming the whole tree from HBM again.
__device__ __forceinline__ void push_tasks(const RetainParams& p, RTask* out, u32* n_out, u32, u32 q, u32 pos, u32 mode, u32 kb, u32 kn) {
    const u32 nt = (kn + RTASK_CHUNK - 1) / RTASK_CHUNK;
    if (nt == 0) return;
    const u32 sq = min(RQ - 1u, static_cast<u32>((static_cast<unsigned long long>(kb) * RQ) / max(p.v.n_kids, 1u)));
    const u32 at = atomicAdd(n_out + sq, nt);
    // on overflow the lookup is retried with a larger scratch, but the next round of THIS attempt still reads the slice up to
    // cap_items: the tasks that fit are stored, so that it never reads an entry nobody wrote
    const u32 fit = at < p.cap_items ? min(nt, p.cap_items - at) : 0u;
    if (fit < nt) atomicOr(p.err, 1u);
    RTask* dst = out + static_cast<size_t>(sq) * p.cap_items + at;
    for (u32 j = 0; j < fit; ++j) dst[j] = RTask{q, pos | (mode << 30), kb + j * RTASK_CHUNK, min(RTASK_CHUNK, kn - j * RTASK_CHUNK)};
}

// The record of the node a thread currently stands on.  `mask`: 32-bit Bloom mask over the tokens of its children (it
// travels in the spare word of the parent's child-block entry; all ones when the record came from a hash slot, which
// has no spare word): a clear bit proves the exact child does not exist and saves the probe — after a '+' expansion
// most children do NOT continue the filter's next literal level.
struct RRec { u32 node, first_kid, nk_flags, val, val_lo, val_hi, mask; };

// RetainTree::_matches (retain.rs:298-367) from node `r` at filter position `pos`, following exact levels in place.
// SMALL child blocks are expanded IN PLACE: a '+' (or a shadowed '#') at a node with at most RINLINE_KIDS children loops over
// them right here (explicit stack of RINLINE_DEPTH frames) instead of becoming a task for the next round — measured on C4,
// 838 K of the 1.02 M tasks of a batch had 1..5 children (a device's sensors, a sensor's metrics), and a task costs a
// queue record, a warp and ~500 warp-instructions of bookkeeping whatever its size.
constexpr u32 RINLINE_KIDS = 8, RINLINE_DEPTH = 4;
template <bool STATS, bool TTL>
__device__ __forceinline__ void retain_chain(const RetainParams& p, u64 now, RTask* out, u32* n_out, u32 sq, u32 q, u32 L, u32 pos, RRec r,
                                             unsigned long long& visited, unsigned long long& probes) {
    const RetainView& v = p.v;
    u32 st_kb[RINLINE_DEPTH], st_ke[RINLINE_DEPTH], st_pm[RINLINE_DEPTH];     // child range still to visit, pos | mode << 30
    u32 sp = 0;
    for (;;) {
        // ---- one node: `r` at filter position `pos` ----
        bool descend = false;
        do {
            if (STATS) ++visited;
            const u32 nkids = r.nk_flags & RNK_MASK, flags = r.nk_flags >> 28;
            if (nkids == 0 || pos == L) {                                        // retain.rs:305-311
                if (pos == L && (flags & 8u)) emit_value<TTL>(p, now, sq, q, r.val);
                break;
            }
            const u32 tok = retain_tok(p, q, pos);
            const bool next_hash = (pos + 1 < L) && retain_tok(p, q, pos + 1) == TOK_HASH;
            // precise matching first — Level equality, so a stored literal "+" / "#" child shadows the wildcard
            // expansion (retain.rs:313)
            const bool exact_try = tok >= TOK_BLANK || (tok == TOK_PLUS && (flags & RF_LIT_PLUS)) || (tok == TOK_HASH && (flags & RF_LIT_HASH));
            u32 c[8];
            bool found = false;
            if (exact_try && (r.mask & retain_mask_bit(tok))) { if (STATS) ++probes; found = retain_child(v, r.node, tok, c); }
            if (found) {
                if (next_hash && ((c[4] >> 28) & 8u)) emit_value<TTL>(p, now, sq, q, c[5]);   // '#' matches the parent, retain.rs:317-322
                r = RRec{c[2], c[3], c[4], c[5], c[6], c[7], 0xFFFFFFFFu};
                ++pos;
                descend = true;
                break;
            }
            const bool root = r.node == 0;
            const u32 nexp = root ? v.root_plain_kids : nkids;
            u32 mode = 0;
            if (tok == TOK_PLUS) mode = 1u;                                       // retain.rs:324-342
            else if (tok == TOK_HASH) {                                           // retain.rs:343-365
                if (!(flags & RF_SUB_LIT_HASH)) {       // every strict descendant (minus `$` subtrees at the root): one range
                    const u32 lo = r.val_lo + ((flags & 8u) ? 1u : 0u), hi = root ? v.root_plain_val_hi : r.val_hi;
                    if (hi > lo) emit_desc(p, sq, q, lo, hi - lo, 1u);
                } else mode = 2u;
            }
            if (mode) {
                if (nexp <= RINLINE_KIDS && sp < RINLINE_DEPTH) { st_kb[sp] = r.first_kid; st_ke[sp] = r.first_kid + nexp; st_pm[sp] = pos | (mode << 30); ++sp; }
                else push_tasks(p, out, n_out, sq, q, pos, mode, r.first_kid, nexp);
            }
        } while (false);
        if (descend) continue;
        // ---- next child of the innermost in-place expansion (same per-child logic as k_retain_round's stage A) ----
        bool have = false;
        while (sp && !have) {
            if (st_kb[sp - 1] == st_ke[sp - 1]) { --sp; continue; }
            u32 kd[8];
            ld256(v.kids + st_kb[sp - 1]++, kd);
            const u32 fpos = st_pm[sp - 1] & 0x3FFFFFFFu, fmode = st_pm[sp - 1] >> 30;
            const bool has_val = ((kd[3] >> 28) & 8u) != 0;
            const u32 kkids = kd[3] & RNK_MASK;
            if (STATS) ++visited;
            if (fmode == 1u) {
                if (fpos + 1 == L) { if (has_val) emit_value<TTL>(p, now, sq, q, kd[4]); continue; }
                if (has_val && (fpos + 1 < L) && retain_tok(p, q, fpos + 1) == TOK_HASH) emit_value<TTL>(p, now, sq, q, kd[4]);   // `.../+/#` parent match
                if (!kkids) continue;
                pos = fpos + 1;
            } else {
                if (has_val) emit_value<TTL>(p, now, sq, q, kd[4]);
                if (!kkids) continue;
                pos = fpos;
            }
            r = RRec{kd[1], kd[2], kd[3], kd[4], kd[5], kd[6], kd[7]};
            have = true;
        }
        if (!have) return;
    }
}

// round 0: one thread per query walks the literal prefix of its filter from the root
template <bool STATS, bool TTL>
__global__ void __launch_bounds__(256)
k_retain_init(RetainParams p, RTask* out, u32* n_out) {
    const u32 q = blockIdx.x * blockDim.x + threadIdx.x;
    const u32 n_act = p.n_ptr ? min(p.nq, *p.n_ptr) : p.nq;
    const u64 now = TTL ? *p.now : 0ull;
    unsigned long long visited = 0, probes = 0;
    if (q < n_act) {
        const u32 m = p.qmeta[q];
        if (!(m & META_INVALID))
            retain_chain<STATS, TTL>(p, now, out, n_out, (q >> 5) % RQ, q, m & META_NLEV_MASK, 0u,
                                RRec{0u, p.v.root_first_kid, p.v.root_nk_flags, 0u, 0u, p.v.root_plain_val_hi, 0xFFFFFFFFu}, visited, probes);
    }
    if (STATS && (visited | probes)) { atomicAdd(p.stats, visited); atomicAdd(p.stats + 1, probes); }
}

// round r >= 1: one warp per task.  The child block is read coalesced (32 entries = 1 KB per step), every lane takes one
// child.  What follows below a child is a run of EXACT filter levels, the same for every child of the task — so the
// warp walks it in LOCK STEP instead of lane by lane: children whose Bloom mask admits the next level are compacted
// (ballot) into a per-warp list of node ids in shared memory; the list is then probed 32 nodes per instruction, the
// nodes that exist and go on form the next list, and so on down the exact run.  Every probe instruction therefore has
// (nearly) all 32 lanes busy and 32 independent random loads in flight, where a lane-by-lane walk leaves most lanes
// idle and few loads in flight.  Anything that is not an exact level (the next '+', a '#', a stored literal wildcard) goes through retain_chain as before.
constexpr u32 RLIST = 256;    // = RTASK_CHUNK: at most one survivor per child of the task
#ifndef GM_RETAIN_CTAS
#define GM_RETAIN_CTAS 6
#endif
template <bool STATS, bool TTL>
__global__ void __launch_bounds__(256, GM_RETAIN_CTAS)
k_retain_round(RetainParams p, const RTask* __restrict__ in, const u32* __restrict__ n_in_p, RTask* __restrict__ out, u32* n_out, u32* __restrict__ claim) {
    static_assert(RLIST >= RTASK_CHUNK, "the survivor list holds one entry per child of a task");
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, lt = lanemask_lt();
    const u32 gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    const RetainView& v = p.v;
    __shared__ u32 s_pre[RQ + 1];
    __shared__ u32 s_list[8][2][RLIST];
    const u32 n_in = queue_prefix(n_in_p, p.cap_items, s_pre);
    const u64 now = TTL ? *p.now : 0ull;
    const u32 sq = gwarp % RQ;                        // this warp appends to its own slice
    unsigned long long visited = 0, probes = 0;
    // tasks differ in size by two orders of magnitude (1 .. 256 children, 0 .. 3 probe levels below): warps CLAIM them one
    // at a time from a shared counter instead of taking a fixed stride
    (void)nwarps;
    for (;;) {
        u32 ti = 0;
        if (lane == 0) ti = atomicAdd(claim, 1u);
        ti = __shfl_sync(0xFFFFFFFFu, ti, 0);
        if (ti >= n_in) break;
        const uint4 tw = *reinterpret_cast<const uint4*>(in + queue_locate(s_pre, ti, p.cap_items));
        const u32 q = tw.x, pos = tw.y & 0x3FFFFFFFu, mode = tw.y >> 30, kb = tw.z, kn = tw.w;
        const u32 L = p.qmeta[q] & META_NLEV_MASK;
        const bool next_hash = mode == 1u && (pos + 1 < L) && retain_tok(p, q, pos + 1) == TOK_HASH;
        // the filter position the children continue at, and the level found there (uniform over the warp)
        u32 P = mode == 1u ? pos + 1 : pos;
        u32 tokP = P < L ? retain_tok(p, q, P) : TOK_UNKNOWN;
        u32 cur = 0, cnt = 0;
        // ---- stage A: the children ----
        for (u32 e0 = 0; e0 < kn; e0 += 32) {
            const u32 e = e0 + lane;
            bool want = false;
            u32 wnode = 0;
            if (e < kn) {
                u32 kd[8];                                          // {token, child, first_kid, nk_flags, val, val_lo, val_hi, child-token mask}
                ld256(v.kids + kb + e, kd);
                if (STATS) ++visited;
                const bool has_val = ((kd[3] >> 28) & 8u) != 0;
                const u32 kkids = kd[3] & RNK_MASK;
                bool go = false;
                if (mode == 1u) {
                    if (pos + 1 == L) { if (has_val) emit_value<TTL>(p, now, sq, q, kd[4]); }   // filter ends here: the child's own value
                    else {
                        if (next_hash && has_val) emit_value<TTL>(p, now, sq, q, kd[4]);        // `.../+/#` parent match
                        go = kkids != 0;
                    }
                } else {                                            // '#' one level at a time (a literal "#" child hides below)
                    if (has_val) emit_value<TTL>(p, now, sq, q, kd[4]);
                    go = kkids != 0;
                }
                if (go) {
                    if (tokP >= TOK_BLANK) { want = (kd[7] & retain_mask_bit(tokP)) != 0; wnode = kd[1]; }   // exact level: lock-step list
                    else retain_chain<STATS, TTL>(p, now, out, n_out, sq, q, L, P, RRec{kd[1], kd[2], kd[3], kd[4], kd[5], kd[6], kd[7]}, visited, probes);
                }
            }
            const u32 bal = __ballot_sync(0xFFFFFFFFu, want);
            if (want) s_list[wid][cur][cnt + __popc(bal & lt)] = wnode;
            cnt += __popc(bal);
        }
        // ---- stage B: down the run of exact levels, 32 nodes per probe instruction ----
        while (cnt) {                                               // (uniform: cnt, P, tokP are warp-wide values)
            const bool nh = (P + 1 < L) && retain_tok(p, q, P + 1) == TOK_HASH;
            const u32 P1 = P + 1;
            const u32 tok1 = P1 < L ? retain_tok(p, q, P1) : TOK_UNKNOWN;
            u32 ncnt = 0;
            __syncwarp();
            for (u32 b0 = 0; b0 < cnt; b0 += 32) {
                bool want = false;
                u32 wnode = 0;
                if (b0 + lane < cnt) {
                    const u32 node = s_list[wid][cur][b0 + lane];
                    u32 c[8];
                    if (STATS) { ++probes; ++visited; }
                    if (retain_child(v, node, tokP, c)) {
                        const u32 fl = c[4] >> 28, nk = c[4] & RNK_MASK;
                        if (nh && (fl & 8u)) emit_value<TTL>(p, now, sq, q, c[5]);              // '#' matches the parent, retain.rs:317-322
                        if (nk == 0 || P1 == L) { if (P1 == L && (fl & 8u)) emit_value<TTL>(p, now, sq, q, c[5]); }   // retain.rs:305-311
                        else if (tok1 >= TOK_BLANK) { want = true; wnode = c[2]; }             // another exact level (a hash slot has no mask)
                        else retain_chain<STATS, TTL>(p, now, out, n_out, sq, q, L, P1, RRec{c[2], c[3], c[4], c[5], c[6], c[7], 0xFFFFFFFFu}, visited, probes);
                    }
                }
                const u32 bal = __ballot_sync(0xFFFFFFFFu, want);
                if (want) s_list[wid][cur ^ 1][ncnt + __popc(bal & lt)] = wnode;
                ncnt += __popc(bal);
            }
            cur ^= 1; cnt = ncnt; P = P1; tokP = tok1;
        }
        __syncwarp();
    }
    if (STATS) {
#pragma unroll
        for (int o = 16; o; o >>= 1) { visited += __shfl_xor_sync(0xFFFFFFFFu, visited, o); probes += __shfl_xor_sync(0xFFFFFFFFu, probes, o); }
        if (lane == 0 && (visited | probes)) { atomicAdd(p.stats, visited); atomicAdd(p.stats + 1, probes); }
    }
}

// Exclusive scan of qtotal -> qbase, spans; single block (nq is a batch of SUBSCRIBE filters).  n_ptr (small-batch graphs):
// the real filter count, read from device memory; nq is then the capacity.
__global__ void __launch_bounds__(1024)
k_retain_scan(const u32* __restrict__ qtotal, u32 nq, const u32* __restrict__ n_ptr, u32* __restrict__ qbase, uint2* __restrict__ spans, unsigned long long* grand) {
    __shared__ unsigned long long s_part[1024];
    if (n_ptr) nq = min(nq, *n_ptr);
    const u32 tid = threadIdx.x;
    const u32 per = (nq + 1023) / 1024;
    const u32 b = min(nq, tid * per), e = min(nq, b + per);
    unsigned long long sum = 0;
    for (u32 i = b; i < e; ++i) sum += qtotal[i];
    s_part[tid] = sum;
    __syncthreads();
    if (tid == 0) {
        unsigned long long run = 0;
        for (int i = 0; i < 1024; ++i) { unsigned long long x = s_part[i]; s_part[i] = run; run += x; }
        *grand = run;
    }
    __syncthreads();
    unsigned long long run = s_part[tid];
    for (u32 i = b; i < e; ++i) {
        const u32 c = qtotal[i];
        const u32 off = run > 0xFFFFFFFFull ? 0xFFFFFFFFu : static_cast<u32>(run);
        qbase[i] = off;
        spans[i] = make_uint2(off, c);
        run += c;
    }
}

// lanes [a, b) of a warp (0 <= a <= b <= 32, a < 32)
__device__ __forceinline__ u32 lane_range(u32 a, u32 b) { return (b >= 32 ? 0xFFFFFFFFu : (1u << b) - 1u) & ~((1u << a) - 1u); }

// With deadlines only, between the last round and k_retain_scan: a '#' range descriptor (kind 1) counted every value of its
// range in qtotal.  This pass subtracts the expired ones and keeps the range's live count in the descriptor
// (kind = 1 | live << 1) for k_retain_expand.  Load-balanced like the expansion: a warp takes 32 descriptors and reads their
// ranges 32 values per step; every descriptor's lane counts the expired values of its own run in the step's ballot.
__global__ void __launch_bounds__(256)
k_retain_live(RDesc* __restrict__ descs, const u32* __restrict__ n_desc_p, u32 cap_desc, const u32* __restrict__ rvals, u32* __restrict__ qtotal,
              const u64* __restrict__ dl, u32 n_dl, const u64* __restrict__ now_p) {
    const u32 lane = threadIdx.x & 31;
    const u32 gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    __shared__ u32 s_pre[RQ + 1];
    const u32 nd = queue_prefix(n_desc_p, cap_desc, s_pre);
    const u64 now = *now_p;
    for (u32 base = gwarp * 32; base < nd; base += nwarps * 32) {
        const u32 i = base + lane;
        const size_t at = i < nd ? queue_locate(s_pre, i, cap_desc) : 0;
        const RDesc d = i < nd ? descs[at] : RDesc{0, 0, 0, 0};
        const u32 ni = d.kind == 1u ? d.cnt : 0u;                // single values were checked where they were emitted
        u32 sc = ni;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { u32 x = __shfl_up_sync(0xFFFFFFFFu, sc, o); if (lane >= o) sc += x; }
        const u32 tot = __shfl_sync(0xFFFFFFFFu, sc, 31);
        const u32 exc = sc - ni;
        u32 dead = 0;
        for (u32 e0 = 0; e0 < tot; e0 += 32) {
            const u32 e = e0 + lane;
            const u32 lo = warp_run_owner(exc, e);
            const u32 o_exc = __shfl_sync(0xFFFFFFFFu, exc, lo);
            const u32 o_ref = __shfl_sync(0xFFFFFFFFu, d.ref, lo);
            const bool x = e < tot && !retain_live(dl, n_dl, now, rvals[o_ref + (e - o_exc)]);
            const u32 bal = __ballot_sync(0xFFFFFFFFu, x);
            const u32 a = max(exc, e0), b = min(exc + ni, e0 + 32u);
            if (b > a) dead += __popc(bal & lane_range(a - e0, b - e0));
        }
        __syncwarp();      // no lane leaves before every lane took the last ballot (the CPU emulation drops exited lanes from it)
        if (ni) {
            if (dead) atomicAdd(qtotal + d.q, 0u - dead);       // (modular: subtracts)
            descs[at].kind = 1u | ((ni - dead) << 1);
        }
    }
}

// Expands the descriptors into per-query contiguous lists (load-balanced like the publish step of k_match_fast).  TTL: the
// ranges carry their live count (k_retain_live); expired values are compacted out with a warp ballot, so that every filter's
// handles stay contiguous: a value goes to its descriptor's slot + the live values of its run in earlier steps + the live
// lanes of its run before it in this step.
template <bool TTL>
__global__ void __launch_bounds__(256)
k_retain_expand(const RDesc* __restrict__ descs, const u32* __restrict__ n_desc_p, u32 cap_desc, const u32* __restrict__ rvals,
                const u32* __restrict__ qbase, u32* __restrict__ qcur, u32* __restrict__ out, unsigned long long cap_ids,
                const u64* __restrict__ dl, u32 n_dl, const u64* __restrict__ now_p) {
    const u32 lane = threadIdx.x & 31;
    const u32 gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    __shared__ u32 s_pre[RQ + 1];
    const u32 nd = queue_prefix(n_desc_p, cap_desc, s_pre);
    const u64 now = TTL ? *now_p : 0ull;
    for (u32 base = gwarp * 32; base < nd; base += nwarps * 32) {
        const u32 i = base + lane;
        RDesc d = i < nd ? descs[queue_locate(s_pre, i, cap_desc)] : RDesc{0, 0, 0, 0};
        const u32 ni = d.cnt;
        const u32 nl = TTL && d.kind ? d.kind >> 1 : ni;        // slots to reserve: the live values
        const u32 dst = nl ? qbase[d.q] + atomicAdd(qcur + d.q, nl) : 0u;
        u32 sc = ni;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { u32 x = __shfl_up_sync(0xFFFFFFFFu, sc, o); if (lane >= o) sc += x; }
        const u32 tot = __shfl_sync(0xFFFFFFFFu, sc, 31);
        const u32 exc = sc - ni;
        u32 run = 0;                                             // TTL: live values of this lane's descriptor written so far
        for (u32 e0 = 0; e0 < tot; e0 += 32) {
            const u32 e = e0 + lane;
            const u32 lo = warp_run_owner(exc, e);
            const u32 o_exc = __shfl_sync(0xFFFFFFFFu, exc, lo);
            const u32 o_ref = __shfl_sync(0xFFFFFFFFu, d.ref, lo);
            const u32 o_kind = __shfl_sync(0xFFFFFFFFu, d.kind, lo);
            const u32 o_dst = __shfl_sync(0xFFFFFFFFu, dst, lo);
            if (TTL) {
                const u32 o_run = __shfl_sync(0xFFFFFFFFu, run, lo);
                const u32 k = e - o_exc;
                const u32 v = e < tot ? (o_kind ? rvals[o_ref + k] : o_ref) : 0u;
                const bool live = e < tot && (!o_kind || retain_live(dl, n_dl, now, v));
                const u32 bal = __ballot_sync(0xFFFFFFFFu, live);
                const u32 first = o_exc > e0 ? o_exc - e0 : 0u;    // this run's first lane in the step
                const unsigned long long at = static_cast<unsigned long long>(o_dst) + o_run + __popc(bal & lane_range(first, lane));
                if (live && at < cap_ids) __stcs(out + at, v);
                const u32 a = max(exc, e0), b = min(exc + ni, e0 + 32u);
                if (b > a) run += __popc(bal & lane_range(a - e0, b - e0));
            } else if (e < tot) {
                const u32 k = e - o_exc;
                const unsigned long long at = static_cast<unsigned long long>(o_dst) + k;
                if (at < cap_ids) __stcs(out + at, o_kind ? rvals[o_ref + k] : o_ref);
            }
        }
        if (TTL) __syncwarp();   // as in k_retain_live
    }
}

}  // namespace gm
