// Device-side relation expansion (SURVEY.md §8f-1): what DefaultRouter::_matches does with every matched relation
// AFTER the trie walk (rmqtt/src/router.rs:182-239, rmqtt/src/types.rs:478-508), for a whole batch:
//
//   * `no_local` (router.rs:184-189): a v5 subscriber that set no_local does not receive its own PUBLISH — the relation is
//     dropped when the publisher's Id equals the subscriber's Id;
//   * shared-subscription members (router.rs:192-200) and v3 relations pass through in k_relations<false>; k_relations<true>
//     instead makes the choice of ONE member per group (router.rs:224-238) with a seeded draw;
//   * v5 relations are de-duplicated PER CLIENT (types.rs:488-506): a client that matches through several filters gets ONE
//     relation, and the subscription identifiers of all its matching subscriptions accumulate.
//
// Input: the match kernels' own output (spans + relation handles, device buffers) and a 16-byte record per handle.
// Output: per topic the finished gm_sub_relation records {node id, handle, group, sub-id range} (the reference's SubRelation
// minus the strings the host resolves from the handle) and the accumulated subscription ids.  One warp per topic; the v5 relations of a topic are staged
// in shared memory and de-duplicated by an all-pairs pass (a topic rarely has more than a few dozen); a topic with more
// than REL_STAGE v5 relations is flagged (status 1) and handed to the host un-deduplicated.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>

#include "../../include/gpumqtt.h"
#include "kernels.cuh"

namespace gm {

constexpr u32 REL_STAGE = 256;
constexpr u32 REL_NONE = 0xFFFFFFFFu;

struct RelParams {
    const uint2* spans; const u32* ids; u32 n;
    const u32* pubs;                 // [n] id_idx of the publisher or REL_NONE; may be null
    const gm_rel* rels; u32 n_rels;
    uint2* out_spans; gm_sub_relation* out_rels; unsigned long long cap_rels;
    u32* out_sub_ids; unsigned long long cap_sub_ids;
    unsigned long long* needed;      // [2] relations, sub ids  ([2] unused)
    int* status;                     // [n]
};

__device__ __forceinline__ u32 warp_incl_scan(u32 v, u32 lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const u32 x = __shfl_up_sync(0xFFFFFFFFu, v, o); if (lane >= o) v += x; }
    return v;
}

__device__ __forceinline__ gm_rel load_rel(const gm_rel* p) {      // 24-byte record, 8-byte aligned
    const uint2* q = reinterpret_cast<const uint2*>(p);
    const uint2 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2);
    gm_rel r;
    r.node_id = (static_cast<unsigned long long>(a.y) << 32) | a.x; r.client_key = b.x; r.id_idx = b.y; r.sub_id = c.x; r.flags = c.y;
    return r;
}

// ---- shared subscriptions: ONE member per (matched filter, group) and appearance (router.rs:192-238, subscribe.rs:66-104) ----
// The reference draws with rand::random; here the draw is a random-key minimum that is deterministic given a seed and does not
// depend on member order: every eligible member gets key = share_key(seed, row, group, occ, client_key), and the chosen one is
// the ONLINE eligible member with the smallest (key, client_key), else the smallest of all eligible members, flagged offline.
// That is uniform over the online members, otherwise over all of them — the reference's distribution.  `occ` numbers the
// appearances of the group in one row (a topic with a literal '+' / '#' level matches a wildcard filter node twice, and the
// reference then runs the choice twice, router.rs:166).
__host__ __device__ __forceinline__ unsigned long long share_mix(unsigned long long x) {
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull; x ^= x >> 27; x *= 0x94d049bb133111ebull; x ^= x >> 31;
    return x;
}
__host__ __device__ __forceinline__ unsigned long long share_key(unsigned long long seed, u32 row, u32 group, u32 occ, u32 client_key) {
    return share_mix(share_mix(seed ^ ((static_cast<unsigned long long>(row) << 32) | group)) ^ ((static_cast<unsigned long long>(occ) << 32) | client_key));
}

struct RelGroups {
    const uint2* groups; u32 n_groups;   // [group id] = {off, cnt}: the group's live member handles in members[]
    const u32* members;
    const u32* online; u32 n_online_bits;   // one bit per client_key; null: every client online
    unsigned long long seed;
};

// (offline, key, client_key, handle) of a candidate; offline = 2 stands for "no candidate"
struct ShareCand { u32 off; unsigned long long key; u32 ck, h; };
__device__ __forceinline__ bool share_less(const ShareCand& a, const ShareCand& b) {
    if (a.off != b.off) return a.off < b.off;
    if (a.key != b.key) return a.key < b.key;
    if (a.ck != b.ck) return a.ck < b.ck;
    return a.h < b.h;
}

// the choice of the whole warp for one appearance of group `grp` in row t; returns the chosen handle (REL_NONE: no eligible
// member), warp-uniform.  Eligible = live and not dropped by no_local (router.rs:184-189 runs before the bucketing).
__device__ __forceinline__ u32 share_choose(const RelParams& p, const RelGroups& g, u32 t, u32 grp, u32 occ, u32 pub, u32 lane, bool& offline) {
    const uint2 blk = g.groups[grp];
    ShareCand best{2u, 0ull, 0u, REL_NONE};
    for (u32 m0 = 0; m0 < blk.y; m0 += 32) {
        const u32 m = m0 + lane;
        if (m >= blk.y) break;
        const u32 h = g.members[blk.x + m];
        if (h >= p.n_rels) continue;
        const gm_rel r = load_rel(p.rels + h);
        if (!(r.flags & GM_REL_LIVE)) continue;
        if ((r.flags & GM_REL_V5) && (r.flags & GM_REL_NO_LOCAL) && pub != REL_NONE && r.id_idx == pub) continue;
        const u32 ck = r.client_key;
        const u32 off = g.online && (ck >= g.n_online_bits || !((g.online[ck >> 5] >> (ck & 31u)) & 1u)) ? 1u : 0u;
        const ShareCand c{off, share_key(g.seed, t, grp, occ, ck), ck, h};
        if (share_less(c, best)) best = c;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const ShareCand c{__shfl_xor_sync(0xFFFFFFFFu, best.off, o), __shfl_xor_sync(0xFFFFFFFFu, best.key, o),
                          __shfl_xor_sync(0xFFFFFFFFu, best.ck, o), __shfl_xor_sync(0xFFFFFFFFu, best.h, o)};
        if (share_less(c, best)) best = c;
    }
    offline = best.off == 1u;
    return best.h;
}

// Choose = false: every shared member passes through as a record of its own (group field = its group id); `g` is unused.
// Choose = true: in a row's match list a shared member stands for its group only if it is the group's REPRESENTATIVE
// (members[groups[g].off]); every other member entry is dropped.  Every matched filter node emits its whole value set, so the
// representative appears once per appearance of the group.  Per appearance the warp scans the group's block and chooses; a
// chosen v3 member is a direct record, a chosen v5 member joins the row's v5 relations and is de-duplicated per client with
// them.  A chosen record's group field is the group id | GM_SUBREL_OFFLINE when it was chosen offline.
// In both forms a de-duplicated v5 record carries the client's smallest handle and that handle's group field.  The choosing
// form alone stages the group fields (s_grp): the expand form keeps 24 KiB of shared memory and its registers.
// k_relations(p) is the expand form; k_relations_choose (below) names the choosing one.
template <bool Choose = false>
__global__ void __launch_bounds__(256)
k_relations(RelParams p, RelGroups g = RelGroups{}) {
    __shared__ u32 s_key[8][REL_STAGE], s_h[8][REL_STAGE], s_sub[8][REL_STAGE], s_grp[8][Choose ? REL_STAGE : 1];
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, lt = lanemask_lt();
    const u32 gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    u32* sk = s_key[wid]; u32* sh = s_h[wid]; u32* ss = s_sub[wid]; u32* sg = s_grp[wid];
    for (u32 t = gwarp; t < p.n; t += nwarps) {
        const uint2 sp = p.spans[t];
        const u32 off = sp.x, cnt = sp.y;
        const u32 pub = p.pubs ? p.pubs[t] : REL_NONE;
        // classify one handle: 0 dropped, 1 direct (v3, or a shared member passed through), 2 v5 relation subject to per-client
        // de-dup, 3 a group's representative (choosing form)
        auto classify = [&](u32 i, u32& h, gm_rel& r) -> u32 {
            if (i >= cnt) return 0u;
            h = p.ids[off + i];
            if (h >= p.n_rels) return 0u;
            r = load_rel(p.rels + h);
            if (!(r.flags & GM_REL_LIVE)) return 0u;
            const u32 grp = r.flags >> 8;
            if constexpr (Choose) if (grp) return grp < g.n_groups && g.groups[grp].y && g.members[g.groups[grp].x] == h ? 3u : 0u;   // no_local: in the choice
            if ((r.flags & GM_REL_V5) && (r.flags & GM_REL_NO_LOCAL) && pub != REL_NONE && r.id_idx == pub) return 0u;   // router.rs:184-189
            return ((r.flags & GM_REL_V5) && grp == 0u) ? 2u : 1u;
        };
        // the choices of the representatives in one 32-entry chunk, in list order; f(handle, record, group field) per chosen member
        auto each_choice = [&](u32 i0, u32 c, u32 h, u32 grp, auto&& f) {
            if constexpr (Choose) {
                u32 bt = __ballot_sync(0xFFFFFFFFu, c == 3u);
                while (bt) {
                    const u32 src = __ffs(bt) - 1; bt &= bt - 1;
                    const u32 rh = __shfl_sync(0xFFFFFFFFu, h, src), rg = __shfl_sync(0xFFFFFFFFu, grp, src), at = i0 + src;
                    u32 occ = 0;                                            // earlier appearances of the same representative
                    for (u32 j0 = 0; j0 < at; j0 += 32) occ += __popc(__ballot_sync(0xFFFFFFFFu, j0 + lane < at && p.ids[off + j0 + lane] == rh));
                    bool offline = false;
                    const u32 ch = share_choose(p, g, t, rg, occ, pub, lane, offline);
                    if (ch != REL_NONE) f(ch, load_rel(p.rels + ch), rg | (offline ? GM_SUBREL_OFFLINE : 0u));
                }
            }
        };
        // ---- pass 1: count, choose, stage the v5 relations (chosen v5 members included) ----
        u32 ndirect = 0, nv = 0;
        for (u32 i0 = 0; i0 < cnt; i0 += 32) {
            u32 h = 0; gm_rel r{};
            const u32 c = classify(i0 + lane, h, r);
            ndirect += __popc(__ballot_sync(0xFFFFFFFFu, c == 1u));
            const u32 bv = __ballot_sync(0xFFFFFFFFu, c == 2u);
            if (c == 2u) {
                const u32 at = nv + __popc(bv & lt);
                if (at < REL_STAGE) { sk[at] = r.client_key; sh[at] = h; ss[at] = r.sub_id; if constexpr (Choose) sg[at] = 0u; }
            }
            nv += __popc(bv);
            each_choice(i0, c, h, r.flags >> 8, [&](u32 ch, const gm_rel& cr, u32 gw) {
                if (!(cr.flags & GM_REL_V5)) { ++ndirect; return; }
                if (lane == 0 && nv < REL_STAGE) { sk[nv] = cr.client_key; sh[nv] = ch; ss[nv] = cr.sub_id; sg[nv] = gw; }
                ++nv;
            });
        }
        __syncwarp();
        const bool overflow = nv > REL_STAGE;
        // ---- de-dup: entry e represents its client iff it holds the smallest handle of the client's relations (the same handle can
        //      occur twice: a topic with a literal '+' / '#' level visits a wildcard child twice — ties go to the earlier entry) ----
        u32 nreps = 0, nsubs = 0;
        if (!overflow) {
            for (u32 e0 = 0; e0 < nv; e0 += 32) {
                const u32 e = e0 + lane;
                bool rep = false; u32 nsub = 0;
                if (e < nv) {
                    const u32 key = sk[e], h = sh[e];
                    rep = true;
                    for (u32 j = 0; j < nv; ++j) if (sk[j] == key) { rep &= !(sh[j] < h || (sh[j] == h && j < e)); nsub += ss[j] != 0u; }
                }
                nreps += __popc(__ballot_sync(0xFFFFFFFFu, rep));
                nsubs += __reduce_add_sync(0xFFFFFFFFu, rep ? nsub : 0u);
            }
        } else nreps = nv;                       // handed over un-deduplicated
        const u32 total = ndirect + nreps;
        unsigned long long hb = 0, sb = 0;
        if (lane == 0) {
            if (total) hb = atomicAdd(p.needed + 0, static_cast<unsigned long long>(total));
            if (nsubs) sb = atomicAdd(p.needed + 1, static_cast<unsigned long long>(nsubs));
        }
        hb = __shfl_sync(0xFFFFFFFFu, hb, 0); sb = __shfl_sync(0xFFFFFFFFu, sb, 0);
        const bool fits = hb + total <= p.cap_rels && sb + nsubs <= p.cap_sub_ids && hb + total <= 0xFFFFFFFFull && sb + nsubs <= 0xFFFFFFFFull;
        if (lane == 0) { p.out_spans[t] = make_uint2(fits ? static_cast<u32>(hb) : 0u, total); if (overflow) p.status[t] = 1; }
        if (!fits || total == 0) { __syncwarp(); continue; }
        // ---- pass 2: direct records (chosen v3 members; after an overflow every v5 relation too), then the v5 representatives.
        //      The choices are made again: they are a pure function of the row, the group and the appearance ----
        u32 w = 0;
        for (u32 i0 = 0; i0 < cnt; i0 += 32) {
            u32 h = 0; gm_rel r{};
            const u32 c = classify(i0 + lane, h, r);
            const bool take = c == 1u || (overflow && c == 2u);
            const u32 b = __ballot_sync(0xFFFFFFFFu, take);
            if (take) p.out_rels[hb + w + __popc(b & lt)] = gm_sub_relation{r.node_id, h, r.flags >> 8, 0u, 0u};
            w += __popc(b);
            each_choice(i0, c, h, r.flags >> 8, [&](u32 ch, const gm_rel& cr, u32 gw) {
                if ((cr.flags & GM_REL_V5) && !overflow) return;
                if (lane == 0) p.out_rels[hb + w] = gm_sub_relation{cr.node_id, ch, gw, 0u, 0u};
                ++w;
            });
        }
        if (!overflow) {
            u32 ws = 0;
            for (u32 e0 = 0; e0 < nv; e0 += 32) {
                const u32 e = e0 + lane;
                bool rep = false; u32 nsub = 0, key = 0, h = 0;
                if (e < nv) {
                    key = sk[e]; h = sh[e];
                    rep = true;
                    for (u32 j = 0; j < nv; ++j) if (sk[j] == key) { rep &= !(sh[j] < h || (sh[j] == h && j < e)); nsub += ss[j] != 0u; }
                }
                const u32 br = __ballot_sync(0xFFFFFFFFu, rep);
                const u32 mys = rep ? nsub : 0u;
                const u32 inc = warp_incl_scan(mys, lane);
                if (rep) {
                    const u32 so = static_cast<u32>(sb) + ws + (inc - mys);
                    p.out_rels[hb + w + __popc(br & lt)] = gm_sub_relation{load_rel(p.rels + h).node_id, h, Choose ? sg[e] : 0u, nsub ? so : 0u, nsub};
                    u32 k = 0;
                    for (u32 j = 0; j < nv && k < nsub; ++j) if (sk[j] == key && ss[j] != 0u) p.out_sub_ids[so + k++] = ss[j];   // types.rs:497-503
                }
                w += __popc(br); ws += __shfl_sync(0xFFFFFFFFu, inc, 31);
            }
        }
        __syncwarp();
    }
}

constexpr auto k_relations_choose = k_relations<true>;

// One launch of k_relations over the ABI's buffers (n >= 1): the expand form without a group table, the choosing form with
// one.  One warp per topic, at most 8 CTAs per SM.  The caller zeroes o.d_needed first.
inline void launch_relations(const gm_span* spans, const u32* ids, u64 n, const u32* pubs, const gm_rel* rels, u64 n_rels, const gm_rel_groups* gr,
                             const gm_rel_out& o, int num_sms, cudaStream_t s) {
    RelParams rp{};
    rp.spans = reinterpret_cast<const uint2*>(spans); rp.ids = ids; rp.n = static_cast<u32>(n); rp.pubs = pubs;
    rp.rels = rels; rp.n_rels = static_cast<u32>(n_rels);
    rp.out_spans = reinterpret_cast<uint2*>(o.d_spans); rp.out_rels = o.d_rels; rp.cap_rels = o.cap_rels;
    rp.out_sub_ids = o.d_sub_ids; rp.cap_sub_ids = o.cap_sub_ids;
    rp.needed = reinterpret_cast<unsigned long long*>(o.d_needed); rp.status = o.d_status;
    RelGroups rg{};
    if (gr) { rg.groups = reinterpret_cast<const uint2*>(gr->d_groups); rg.n_groups = gr->n_groups; rg.members = gr->d_members; rg.online = gr->d_online; rg.n_online_bits = gr->n_online_bits; rg.seed = gr->seed; }
    const unsigned grid = static_cast<unsigned>(std::min<u64>((n + 7) / 8, static_cast<u64>(num_sms) * 8));
    if (gr) GM_LAUNCH(k_relations_choose, grid, 256, 0, s, rp, rg);
    else GM_LAUNCH(k_relations, grid, 256, 0, s, rp);
}

}  // namespace gm
