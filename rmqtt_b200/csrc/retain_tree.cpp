// Host mirror of the retained-message tree — see retain_tree.h.  Semantics follow
// rmqtt/src/retain.rs:221-257 (insert = value.replace, remove with bottom-up pruning).
#include "retain_tree.h"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <functional>
#include <string_view>

#include "host_par.h"

namespace gm {

int RetainTreeHost::parse(const char* s, u32 len, bool create, std::vector<u32>& toks) {
    return dict_->parse(s, len, create, toks);     // Topic::from_str (topic.rs:348-363)
}

u32 RetainTreeHost::child_of(u32 node, u32 token) const {
    const auto& k = nodes_[node].kids;
    auto it = std::lower_bound(k.begin(), k.end(), std::make_pair(token, 0u));
    return (it != k.end() && it->first == token) ? it->second : 0u;
}

int RetainTreeHost::put(const char* topic, u32 len, u32 value, bool* had_old, u32* old) {
    if (had_old) *had_old = false;
    int st = parse(topic, len, true, toks_);
    if (st != PARSE_OK) return st;
    u32 node = 0;
    bool created = false;
    for (u32 tok : toks_) {
        u32 c = child_of(node, tok);
        if (!c) {
            if (!free_.empty()) { c = free_.back(); free_.pop_back(); nodes_[c] = HN{}; }
            else { c = static_cast<u32>(nodes_.size()); nodes_.emplace_back(); }
            nodes_[c].parent = node; nodes_[c].token = tok;
            auto& k = nodes_[node].kids;
            k.insert(std::lower_bound(k.begin(), k.end(), std::make_pair(tok, 0u)), std::make_pair(tok, c));
            n_nodes_++;
            created = true;
            if (flat_valid_ && (tok == TOK_PLUS || tok == TOK_HASH)) give_up();   // a literal '+' / '#' level changes shadow flags: rebuild
        }
        node = c;
    }
    HN& n = nodes_[node];
    // Re-publishing a retained message on a topic that keeps its handle changes nothing on the device.
    const bool same = n.has_val && n.val == value;
    const bool had = n.has_val;
    if (n.has_val) { if (had_old) *had_old = true; if (old) *old = n.val; }
    else n_values_++;
    n.has_val = true; n.val = value;
    if (same && !created) return PARSE_OK;
    dirty = true;
    if (flat_valid_) dev_set(node, had, value, static_cast<u32>(toks_.size()));
    return PARSE_OK;
}

int RetainTreeHost::remove(const char* topic, u32 len, bool* had_old, u32* old) {
    if (had_old) *had_old = false;
    int st = parse(topic, len, false, toks_);
    if (st != PARSE_OK) return st;
    u32 node = 0;
    for (u32 tok : toks_) {
        if (tok == TOK_UNKNOWN) return PARSE_OK;
        node = child_of(node, tok);
        if (!node) return PARSE_OK;
    }
    HN& n = nodes_[node];
    if (n.has_val) {
        if (had_old) *had_old = true;
        if (old) *old = n.val;
        drop_deadline(n.val);
        n.has_val = false; n.val = RVAL_NONE;
        n_values_--;
        dirty = true;
        if (flat_valid_) dev_unset(node);
    }
    // prune (retain.rs:247-249): value.is_none() && branches.is_empty()
    for (u32 x = node; x != 0;) {
        HN& c = nodes_[x];
        if (c.has_val || !c.kids.empty()) break;
        u32 p = c.parent;
        auto& k = nodes_[p].kids;
        k.erase(std::lower_bound(k.begin(), k.end(), std::make_pair(c.token, 0u)));
        if (flat_valid_) {
            // its device node stays behind as a dead leaf (revived if the path is set again); a literal '+' / '#'
            // level would keep shadowing wildcard expansion -> rebuild
            if (c.token == TOK_PLUS || c.token == TOK_HASH) give_up(); else dead_nodes_++;
        }
        free_.push_back(x);
        n_nodes_--;
        dirty = true;
        x = p;
    }
    return PARSE_OK;
}

int RetainTreeHost::set_ttl(const char* topic, u32 len, u32 value, u64 deadline, bool* had_old, u32* old) {
    if (had_old) *had_old = false;
    if (deadline && value >= DL_MAX_HANDLE) return SET_HANDLE_RANGE;
    if (!dl_topic_.empty()) {
        auto it = dl_topic_.find(value);
        if (it != dl_topic_.end() && std::string_view(it->second) != std::string_view(topic, len)) return SET_CONFLICT;
    }
    bool had = false; u32 o = 0;
    const int st = put(topic, len, value, &had, &o);
    if (st != PARSE_OK) return st;
    if (had_old) *had_old = had;
    if (old && had) *old = o;
    if (had && o != value) drop_deadline(o);
    if (deadline) give_deadline(value, topic, len, deadline); else drop_deadline(value);
    return PARSE_OK;
}

bool RetainTreeHost::holds(const char* topic, u32 len, u32 value) {
    if (parse(topic, len, false, toks_) != PARSE_OK) return false;
    u32 node = 0;
    for (u32 tok : toks_) {
        if (tok == TOK_UNKNOWN) return false;
        if (!(node = child_of(node, tok))) return false;
    }
    return nodes_[node].has_val && nodes_[node].val == value;
}

void RetainTreeHost::give_deadline(u32 h, const char* topic, u32 len, u64 deadline) {
    if (h >= dl.size()) dl.resize(std::max<size_t>({static_cast<size_t>(h) + 1, dl.size() * 2, 1024}), DL_NONE);   // grown: shipped whole
    if (dl[h] != deadline) {
        dl[h] = deadline;
        dirty_dl.push_back(h);
        dl_heap_.emplace_back(deadline, h);
        std::push_heap(dl_heap_.begin(), dl_heap_.end(), std::greater<>());
        dirty = true;
    }
    dl_topic_[h].assign(topic, len);
    if (dl_heap_.size() > 2 * dl_topic_.size() + 4096) {      // mostly stale entries: rebuild from the live deadlines
        dl_heap_.clear();
        for (const auto& kv : dl_topic_) dl_heap_.emplace_back(dl[kv.first], kv.first);
        std::make_heap(dl_heap_.begin(), dl_heap_.end(), std::greater<>());
    }
}

void RetainTreeHost::drop_deadline(u32 h) {
    if (dl_topic_.empty() || !dl_topic_.erase(h)) return;
    dl[h] = DL_NONE;
    dirty_dl.push_back(h);
    dirty = true;
}

int RetainTreeHost::check_batch(const char* blob, const u32* offsets, const u32* values, const u64* deadlines, u64 n) const {
    if (!deadlines && dl_topic_.empty()) return PARSE_OK;
    std::unordered_map<u32, std::pair<bool, std::string_view>> held;   // handle -> (has a deadline, its topic) as the batch goes
    for (u64 i = 0; i < n; ++i) {
        const u32 h = values[i];
        const u64 d = deadlines ? deadlines[i] : 0;
        if (d && h >= DL_MAX_HANDLE) return SET_HANDLE_RANGE;
        const std::string_view t(blob + offsets[i], offsets[i + 1] - offsets[i]);
        auto it = held.find(h);
        if (it == held.end()) {
            auto g = dl_topic_.find(h);
            if (g == dl_topic_.end() && !d) continue;
            it = held.emplace(h, std::make_pair(g != dl_topic_.end(), g != dl_topic_.end() ? std::string_view(g->second) : std::string_view())).first;
        }
        if (it->second.first && it->second.second != t) return SET_CONFLICT;
        it->second = std::make_pair(d != 0, t);
    }
    return PARSE_OK;
}

u64 RetainTreeHost::set_batch_ttl(const char* blob, const u32* offsets, const u32* values, const u64* deadlines, u64 n) {
    const u64 ok = set_batch(blob, offsets, values, n);      // (into an empty tree: the parallel build) — clears replaced deadlines
    std::vector<u32> with;
    for (u64 i = 0; i < n; ++i) if (deadlines[i]) with.push_back(values[i]);
    if (with.empty()) return ok;
    std::sort(with.begin(), with.end());
    for (u64 i = 0; i < n; ++i) {        // in order, as n set_ttl calls: the last entry of a (topic, handle) the tree holds decides
        const u32 h = values[i];
        if (!deadlines[i] && !std::binary_search(with.begin(), with.end(), h)) continue;
        const char* t = blob + offsets[i];
        const u32 len = offsets[i + 1] - offsets[i];
        if (!holds(t, len, h)) continue;
        if (deadlines[i]) give_deadline(h, t, len, deadlines[i]); else drop_deadline(h);
    }
    return ok;
}

u64 RetainTreeHost::remove_expired(u64 now, u32* out, u64 cap) {
    u64 n = 0;
    while (n < cap && !dl_heap_.empty() && dl_heap_.front().first <= now) {
        std::pop_heap(dl_heap_.begin(), dl_heap_.end(), std::greater<>());
        const auto [d, h] = dl_heap_.back();
        dl_heap_.pop_back();
        auto it = dl_topic_.find(h);
        if (it == dl_topic_.end() || dl[h] != d) continue;   // re-set or removed since it was queued
        const std::string topic = it->second;
        bool had = false; u32 old = 0;
        remove(topic.data(), static_cast<u32>(topic.size()), &had, &old);    // drops the deadline
        if (had) out[n++] = old;
    }
    return n;
}

u64 RetainTreeHost::set_batch(const char* blob, const u32* offsets, const u32* values, u64 n) {
    if (nodes_.size() == 1 && free_.empty() && n >= host_par_min(1u << 16) && host_threads() > 1 && !getenv("GM_BULK_SERIAL"))
        return set_batch_build(blob, offsets, values, n, host_threads());
    u64 ok = 0;
    for (u64 i = 0; i < n; ++i)
        if (set(blob + offsets[i], offsets[i + 1] - offsets[i], values[i], nullptr, nullptr) == PARSE_OK) ok++;
    return ok;
}

// Bulk build into an empty tree.  Result: exactly the host tree n calls of set() build and exactly the device image
// flatten() makes of it (same arrays, entry for entry; only the placement of colliding entries inside the hash table depends
// on the thread interleaving) — built without the per-topic walks and without the serial pre-order traversal:
//   1  topics -> tokens on all threads (HostTrie::tokenize_batch, the dictionary is shared with the subscription trie);
//   2  one pass per level: the keys (parent node of the level above, token) of all topics are sorted and made unique — the
//      nodes of the level, in the order flatten() visits the children of a node (root children: plain before `$`);
//   3  bottom-up: subtree sizes, value counts, literal-'#' flags; top-down: pre-order numbers and value ranges (the
//      pre-order number of a child = its parent's + 1 + the sizes of its earlier siblings);
//   4  every node writes its records at its pre-order position; the (parent, token) hash table is filled with CAS claims.
u64 RetainTreeHost::set_batch_build(const char* blob, const u32* offsets, const u32* values, u64 n, unsigned T) {
    const bool prof = getenv("GM_BULK_PROFILE") != nullptr;
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = now();
    HostTrie::TokenizedBatch tb;
    dict_->tokenize_batch(blob, offsets, n, T, tb);
    const double t1 = now();
    u32 deepest = 0;
    u64 n_ok = 0;
    for (u64 i = 0; i < n; ++i) { deepest = std::max<u32>(deepest, tb.depth[i]); n_ok += tb.depth[i] != 0; }
    if (n > 0xFFFFFFF0ull) { fprintf(stderr, "gpumqtt: retained bulk load of more than 2^32 topics\n"); std::abort(); }

    // ---- 2: levels.  lev[0] = {root}; lev[d + 1] = nodes of depth d + 1
    struct Level {
        BigVec<u32> parent, tok;               // index in the level above; level token
        BigVec<u32> last;                      // topic index + 1 of the LAST topic that ends here (value.replace), 0 = none
        BigVec<u32> kid0, nkid;                // children: [kid0, kid0 + nkid) of the level below
        BigVec<u32> size, vcnt, pre, vlo;      // subtree nodes / values, pre-order number, first value slot
        BigVec<u8> sub;                        // RF_SUB_LIT_HASH
        size_t n() const { return parent.size(); }
    };
    std::vector<Level> lev(deepest + 1);
    lev[0].parent.assign(1, 0u); lev[0].tok.assign(1, 0u); lev[0].last.assign(1, 0u);
    BigVec<u32> cur(n, 0u);
    {
        std::vector<std::vector<std::pair<u64, u32>>> pairs(T);
        std::vector<std::vector<u64>> lkeys(T);
        std::vector<u64> ukeys;
        for (u32 d = 0; d < deepest; ++d) {
            parallel_chunks(n, T, [&](unsigned tid, size_t b, size_t e) {
                std::vector<std::pair<u64, u32>> pr; std::vector<u64> lk;
                pr.swap(pairs[tid]); lk.swap(lkeys[tid]);
                pr.clear(); lk.clear();
                for (size_t i = b; i < e; ++i) {
                    if (tb.depth[i] <= d) continue;
                    const u32 tok = tb.toks[tb.lvl_off[i] + d];
                    const u32 key_lo = d == 0 && dict_->token_is_dollar(tok) ? (tok | 0x80000000u) : tok;   // root children: plain first, `$...` last
                    pr.emplace_back((static_cast<u64>(cur[i]) << 32) | key_lo, static_cast<u32>(i));
                }
                std::sort(pr.begin(), pr.end());
                for (size_t k = 0; k < pr.size(); ++k) if (k == 0 || pr[k].first != pr[k - 1].first) lk.push_back(pr[k].first);
                pr.swap(pairs[tid]); lk.swap(lkeys[tid]);
            });
            merge_sorted_unique(lkeys, T, ukeys);
            Level& L = lev[d + 1];
            const size_t nl = ukeys.size();
            if (nl > 0xFFFFFFF0ull) { fprintf(stderr, "gpumqtt: retained bulk load exceeds 2^32 nodes per level\n"); std::abort(); }
            L.parent.resize(nl); L.tok.resize(nl); L.last.assign(nl, 0u);
            parallel_chunks(nl, T, [&](unsigned, size_t b, size_t e) {
                for (size_t g = b; g < e; ++g) { L.parent[g] = static_cast<u32>(ukeys[g] >> 32); L.tok[g] = static_cast<u32>(ukeys[g]) & 0x7FFFFFFFu; }
            });
            // every topic learns its node of this level: its thread's pairs and the level are both sorted by key
            parallel_threads(T, [&](unsigned tid) {
                const auto& pr = pairs[tid];
                if (pr.empty()) return;
                size_t g = static_cast<size_t>(std::lower_bound(ukeys.begin(), ukeys.end(), pr[0].first) - ukeys.begin());
                for (size_t k = 0; k < pr.size(); ++k) {
                    while (ukeys[g] != pr[k].first) ++g;
                    const u32 i = pr[k].second;
                    cur[i] = static_cast<u32>(g);
                    if (tb.depth[i] == d + 1) {             // the topic ends here; of several, the last one's value stays
                        u32 seen = __atomic_load_n(&L.last[g], __ATOMIC_RELAXED);
                        while (seen < i + 1 && !__atomic_compare_exchange_n(&L.last[g], &seen, i + 1, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
                    }
                }
            });
        }
    }
    const double t2 = now();
    // ---- 3: children blocks, bottom-up sums, top-down numbers
    const u32 NL = deepest + 1;
    for (u32 d = 0; d < NL; ++d) {
        Level& L = lev[d];
        L.kid0.assign(L.n(), 0u); L.nkid.assign(L.n(), 0u);
        if (d + 1 < NL) {
            const Level& C = lev[d + 1];
            const size_t nc = C.n();
            BigVec<u32> kend(L.n(), 0u);
            parallel_chunks(nc, T, [&](unsigned, size_t b, size_t e) {
                for (size_t g = b; g < e; ++g) {
                    if (g == 0 || C.parent[g] != C.parent[g - 1]) L.kid0[C.parent[g]] = static_cast<u32>(g);
                    if (g + 1 == nc || C.parent[g + 1] != C.parent[g]) kend[C.parent[g]] = static_cast<u32>(g + 1);
                }
            });
            parallel_chunks(L.n(), T, [&](unsigned, size_t b, size_t e) { for (size_t g = b; g < e; ++g) L.nkid[g] = kend[g] - L.kid0[g]; });
        }
    }
    for (u32 d = NL; d-- > 0;) {
        Level& L = lev[d];
        L.size.resize(L.n()); L.vcnt.resize(L.n()); L.sub.resize(L.n());
        const Level* C = d + 1 < NL ? &lev[d + 1] : nullptr;
        parallel_chunks(L.n(), T, [&](unsigned, size_t b, size_t e) {
            for (size_t g = b; g < e; ++g) {
                u32 sz = 1, vc = L.last[g] ? 1u : 0u; u8 sub = 0;
                for (u32 j = 0; j < L.nkid[g]; ++j) {
                    const u32 c = L.kid0[g] + j;
                    sz += C->size[c]; vc += C->vcnt[c]; sub |= C->sub[c];
                    if (C->tok[c] == TOK_HASH) sub = 1;
                }
                L.size[g] = sz; L.vcnt[g] = vc; L.sub[g] = sub;
            }
        });
    }
    const u64 total_nodes = lev[0].size[0];
    if (total_nodes > 0xFFFFFFF0ull) { fprintf(stderr, "gpumqtt: retained bulk load exceeds 2^32 nodes\n"); std::abort(); }
    for (u32 d = 0; d < NL; ++d) { lev[d].pre.resize(lev[d].n()); lev[d].vlo.resize(lev[d].n()); }
    lev[0].pre[0] = 0; lev[0].vlo[0] = 0;
    for (u32 d = 0; d + 1 < NL; ++d) {
        const Level& L = lev[d];
        Level& C = lev[d + 1];
        parallel_chunks(L.n(), T, [&](unsigned, size_t b, size_t e) {
            for (size_t g = b; g < e; ++g) {
                u32 run = L.pre[g] + 1, vrun = L.vlo[g] + (L.last[g] ? 1u : 0u);
                for (u32 j = 0; j < L.nkid[g]; ++j) {
                    const u32 c = L.kid0[g] + j;
                    C.pre[c] = run; C.vlo[c] = vrun;
                    run += C.size[c]; vrun += C.vcnt[c];
                }
            }
        });
    }
    const double t3 = now();
    // ---- 4: the arrays.  first_kid of a node = child entries of all nodes before it in pre-order
    const size_t NN = static_cast<size_t>(total_nodes);
    const size_t room = (NN - 1) + (NN - 1) / 4 + 1024;      // the slack flatten() leaves for in-place edits
    const u64 total_vals = lev[0].vcnt[0];
    rnodes.clear(); rkids.clear(); rvals.clear();
    rnodes.reserve(std::max(room, NN)); rkids.reserve(std::max(room, NN)); rvals.reserve(total_vals);
    rnodes.resize(NN); rkids.resize(NN - 1); rvals.resize(total_vals);
    rparent_.assign(NN, 0u); rtoken_.assign(NN, 0u); rcap_.assign(NN, 0u); in_rvals_.assign(NN, 0);
    rparent_.reserve(room); rtoken_.reserve(room); rcap_.reserve(room); in_rvals_.reserve(room);
    BigVec<u32> fk(NN + 1, 0u);
    for (u32 d = 0; d < NL; ++d) {
        const Level& L = lev[d];
        parallel_chunks(L.n(), T, [&](unsigned, size_t b, size_t e) { for (size_t g = b; g < e; ++g) fk[L.pre[g] + 1] = L.nkid[g]; });
    }
    for (size_t k = 0; k < NN; ++k) fk[k + 1] += fk[k];
    const double t4a = now();
    nodes_.clear();
    nodes_.resize(NN);
    const double t4b = now();
    for (u32 d = 0; d < NL; ++d) {
        const Level& L = lev[d];
        const Level* C = d + 1 < NL ? &lev[d + 1] : nullptr;
        const Level* P = d ? &lev[d - 1] : nullptr;
        parallel_chunks(L.n(), T, [&](unsigned, size_t b, size_t e) {
            for (size_t g = b; g < e; ++g) {
                const u32 me = L.pre[g];
                const bool has = L.last[g] != 0;
                const u32 val = has ? values[L.last[g] - 1] : RVAL_NONE;
                RNode r{};
                r.first_kid = fk[me]; r.nkids = L.nkid[g];
                r.val = val; r.val_lo = L.vlo[g]; r.val_hi = L.vlo[g] + L.vcnt[g];
                r.flags = (has ? 8u : 0u) | (L.sub[g] ? RF_SUB_LIT_HASH : 0u);
                r.sub_end = me + L.size[g];
                HN& h = nodes_[me];
                h.val = val; h.has_val = has; h.token = d ? L.tok[g] : 0u; h.parent = d ? P->pre[L.parent[g]] : 0u; h.dev = me;
                h.kids.reserve(L.nkid[g]);
                for (u32 j = 0; j < L.nkid[g]; ++j) {
                    const u32 c = L.kid0[g] + j, tok = C->tok[c];
                    r.pad |= retain_mask_bit(tok);
                    if (tok == TOK_PLUS) r.flags |= RF_LIT_PLUS;
                    if (tok == TOK_HASH) r.flags |= RF_LIT_HASH | RF_SUB_LIT_HASH;
                    h.kids.emplace_back(tok, C->pre[c]);
                }
                if (d == 0) std::sort(h.kids.begin(), h.kids.end());     // the host tree keeps every child list sorted by token
                rnodes[me] = r;
                rparent_[me] = h.parent; rtoken_[me] = h.token; rcap_[me] = r.nkids; in_rvals_[me] = has ? 1 : 0;
                if (has) rvals[r.val_lo] = val;
            }
        });
    }
    // child entries and hash slots carry the complete record of the child
    const double t4c = now();
    size_t cap = 1024;
    while (cap < rkids.size() * 4) cap <<= 1;
    redges.assign_zero(cap);
    const double t4d = now();
    const u32 emask = static_cast<u32>(cap - 1);
    for (u32 d = 0; d + 1 < NL; ++d) {
        const Level& L = lev[d];
        const Level& C = lev[d + 1];
        parallel_chunks(L.n(), T, [&](unsigned, size_t b, size_t e) {
            for (size_t g = b; g < e; ++g) {
                const u32 me = L.pre[g], f = fk[me];
                for (u32 j = 0; j < L.nkid[g]; ++j) {
                    const u32 cg = L.kid0[g] + j, cdev = C.pre[cg], tok = C.tok[cg];
                    const RNode& c = rnodes[cdev];
                    const u32 nkf = c.nkids | (c.flags << 28);
                    rkids[f + j] = RKid{tok, cdev, c.first_kid, nkf, c.val, c.val_lo, c.val_hi, c.pad};
                    u32 s = redge_hash(me, tok) & emask;
                    for (;; s = (s + 1) & emask) {                  // claim a slot by its `child` word (never 0 for a real child), then fill it
                        u32 expect = 0;
                        if (__atomic_compare_exchange_n(&redges[s].child, &expect, cdev, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) break;
                    }
                    REdge& ed = redges[s];
                    ed.parent = me; ed.token = tok; ed.first_kid = c.first_kid; ed.nk_flags = nkf; ed.val = c.val; ed.val_lo = c.val_lo; ed.val_hi = c.val_hi;
                }
            }
        });
    }
    // ---- bookkeeping as after set() x n + flatten()
    free_.clear();
    n_nodes_ = NN - 1;
    n_values_ = total_vals;
    max_depth = deepest;
    root_plain_kids = 0;
    root_plain_val_hi = static_cast<u32>(total_vals);
    if (NL > 1) {
        const Level& C = lev[1];
        for (size_t c = 0; c < C.n(); ++c) { if (dict_->token_is_dollar(C.tok[c])) { root_plain_val_hi = C.vlo[c]; break; } root_plain_kids++; }
    }
    flat_valid_ = true; full = true; dirty = true;
    dirty_kids.clear(); dirty_edges.clear(); dirty_vals.clear();
    garbage_kids_ = 0; dead_nodes_ = 0;
    live_edges_ = rkids.size();
    flattens++;
    if (prof) fprintf(stderr, "retained bulk build (%u threads): %llu topics -> %zu nodes: tokens %.2f s, levels %.2f s, numbering %.2f s, arrays %.2f s (allocate %.2f, host nodes %.2f, records %.2f, hash table: allocate %.2f, fill %.2f)\n", T, (unsigned long long)n, NN, t1 - t0, t2 - t1, t3 - t2, now() - t3,
                      t4a - t3, t4b - t4a, t4c - t4b, t4d - t4c, now() - t4d);
    return n_ok;
}

// ------------------------------------------------------------------------------------------------
// In-place maintenance of the device image (see retain_tree.h)
u32 RetainTreeHost::edge_slot_of(u32 parent_dev, u32 token) const {
    const u32 mask = static_cast<u32>(redges.size() - 1);
    for (u32 s = redge_hash(parent_dev, token) & mask;; s = (s + 1) & mask) {
        const REdge& e = redges[s];
        if (e.child == 0) return NODEV;
        if (e.parent == parent_dev && e.token == token) return s;
    }
}

void RetainTreeHost::write_record(u32 dev) {
    if (dev == 0) return;                       // the root's record travels in the kernel parameters (rnodes[0])
    const RNode& r = rnodes[dev];
    const u32 pdev = rparent_[dev], tok = rtoken_[dev];
    const RNode& p = rnodes[pdev];
    for (u32 j = 0; j < p.nkids; ++j) {
        RKid& k = rkids[p.first_kid + j];
        if (k.child != dev) continue;
        k.first_kid = r.first_kid; k.nk_flags = r.nkids | (r.flags << 28); k.val = r.val; k.val_lo = r.val_lo; k.val_hi = r.val_hi; k.pad = r.pad;
        dirty_kids.push_back(p.first_kid + j);
        break;
    }
    const u32 s = edge_slot_of(pdev, tok);
    if (s != NODEV) {
        REdge& e = redges[s];
        e.first_kid = r.first_kid; e.nk_flags = r.nkids | (r.flags << 28); e.val = r.val; e.val_lo = r.val_lo; e.val_hi = r.val_hi;
        dirty_edges.push_back(s);
    }
    patches++;
}

void RetainTreeHost::invalidate_ranges(u32 dev) {
    for (u32 x = dev;; x = rparent_[x]) {
        RNode& r = rnodes[x];
        if (r.flags & RF_SUB_LIT_HASH) break;   // invariant: a flagged node has flagged ancestors
        r.flags |= RF_SUB_LIT_HASH;
        write_record(x);
        if (x == 0) break;
    }
}

u32 RetainTreeHost::dev_new_node(u32 parent_dev, u32 token) {
    const u32 dev = static_cast<u32>(rnodes.size());
    RNode r{};
    r.val = RVAL_NONE;
    r.flags = RF_SUB_LIT_HASH;                  // it has no value range of its own
    rnodes.push_back(r);
    rparent_.push_back(parent_dev); rtoken_.push_back(token); rcap_.push_back(0); in_rvals_.push_back(0);
    return dev;
}

bool RetainTreeHost::dev_add_child(u32 pdev, u32 tok, u32 cdev) {
    if ((live_edges_ + 1) * 2 > redges.size()) return false;                // keep the hash table at most half full
    if (rcap_[pdev] == rnodes[pdev].nkids) {                                   // child block full: move it to the end, doubled
        const u32 oldcap = rcap_[pdev], newcap = std::max<u32>(2u, oldcap * 2u);
        if (rkids.size() + newcap > 0xFFFFFFF0ull) return false;
        const u32 nf = static_cast<u32>(rkids.size());
        rkids.resize(rkids.size() + newcap, RKid{0, 0, 0, 0, RVAL_NONE, 0, 0, 0});
        const u32 of = rnodes[pdev].first_kid;
        for (u32 j = 0; j < rnodes[pdev].nkids; ++j) rkids[nf + j] = rkids[of + j];
        garbage_kids_ += oldcap;
        rnodes[pdev].first_kid = nf;
        rcap_[pdev] = newcap;
    }
    RNode& p = rnodes[pdev];
    const RNode& c = rnodes[cdev];
    u32 idx = p.first_kid + p.nkids;
    if (pdev == 0 && !dict_->token_is_dollar(tok)) {                          // root children: plain first, `$...` last
        if (root_plain_kids < p.nkids) { rkids[idx] = rkids[p.first_kid + root_plain_kids]; dirty_kids.push_back(idx); idx = p.first_kid + root_plain_kids; }
        root_plain_kids++;
    }
    rkids[idx] = RKid{tok, cdev, c.first_kid, c.nkids | (c.flags << 28), c.val, c.val_lo, c.val_hi, c.pad};
    dirty_kids.push_back(idx);
    p.nkids++;
    p.pad |= retain_mask_bit(tok);
    const u32 mask = static_cast<u32>(redges.size() - 1);
    u32 s = redge_hash(pdev, tok) & mask;
    while (redges[s].child != 0) s = (s + 1) & mask;
    redges[s] = REdge{pdev, tok, cdev, c.first_kid, c.nkids | (c.flags << 28), c.val, c.val_lo, c.val_hi};
    dirty_edges.push_back(s);
    live_edges_++;
    write_record(pdev);                          // its block moved / grew
    invalidate_ranges(pdev);
    return true;
}

void RetainTreeHost::dev_set(u32 node, bool had, u32 value, u32 depth) {
    // device nodes for the part of the path that is new to the device (top-down)
    std::vector<u32> missing;
    for (u32 x = node; nodes_[x].dev == NODEV && x != 0; x = nodes_[x].parent) missing.push_back(x);
    for (size_t i = missing.size(); i-- > 0 && flat_valid_;) {
        const u32 m = missing[i];
        const u32 pdev = nodes_[nodes_[m].parent].dev, tok = nodes_[m].token;
        const u32 s = edge_slot_of(pdev, tok);
        if (s != NODEV) { nodes_[m].dev = redges[s].child; if (dead_nodes_) dead_nodes_--; }          // a dead leaf left by an earlier prune
        else {
            const u32 cdev = dev_new_node(pdev, tok);
            if (!dev_add_child(pdev, tok, cdev)) { give_up(); return; }
            nodes_[m].dev = cdev;
        }
    }
    if (!flat_valid_) return;
    const u32 dev = nodes_[node].dev;
    RNode& r = rnodes[dev];
    r.val = value;
    if (had) {                                   // value.replace(v): same shape, same ranges
        if (in_rvals_[dev]) { rvals[r.val_lo] = value; dirty_vals.push_back(r.val_lo); }
        write_record(dev);
    } else {
        r.flags |= 8u;
        write_record(dev);
        invalidate_ranges(dev);
    }
    max_depth = std::max(max_depth, depth);
}

void RetainTreeHost::dev_unset(u32 node) {
    const u32 dev = nodes_[node].dev;
    if (dev == NODEV) { give_up(); return; }
    RNode& r = rnodes[dev];
    r.val = RVAL_NONE;
    r.flags &= ~8u;
    in_rvals_[dev] = 0;
    write_record(dev);
    invalidate_ranges(dev);
}

void RetainTreeHost::prepare_flush() {
    if (flat_valid_ && (garbage_kids_ + dead_nodes_) * 4 > rkids.size() + 4096) give_up();     // too much garbage: re-pack
    if (!flat_valid_) flatten();
}

std::vector<u32> RetainTreeHost::used_tokens() const {
    std::vector<u32> out;
    std::vector<u32> todo{0u};
    while (!todo.empty()) {
        const u32 n = todo.back(); todo.pop_back();
        for (const auto& kv : nodes_[n].kids) { if (kv.first >= TOK_FIRST) out.push_back(kv.first); todo.push_back(kv.second); }
    }
    std::sort(out.begin(), out.end());
    out.erase(std::unique(out.begin(), out.end()), out.end());
    return out;
}

void RetainTreeHost::remap_tokens(const std::vector<u32>& remap) {
    std::vector<u32> todo{0u};
    while (!todo.empty()) {
        const u32 n = todo.back(); todo.pop_back();
        for (auto& kv : nodes_[n].kids) {
            if (kv.first >= TOK_FIRST) kv.first = remap[kv.first];
            nodes_[kv.second].token = kv.first;
            todo.push_back(kv.second);
        }
        std::sort(nodes_[n].kids.begin(), nodes_[n].kids.end());
    }
    give_up();                                   // every token in the device image changed
}

void RetainTreeHost::flatten() {
    rnodes.clear(); rkids.clear(); rvals.clear();
    rparent_.clear(); rtoken_.clear(); rcap_.clear(); in_rvals_.clear();
    rparent_.reserve(n_nodes_ + n_nodes_ / 4 + 1024); rtoken_.reserve(n_nodes_ + n_nodes_ / 4 + 1024);
    rcap_.reserve(n_nodes_ + n_nodes_ / 4 + 1024); in_rvals_.reserve(n_nodes_ + n_nodes_ / 4 + 1024);
    // a quarter of slack: in-place edits append device nodes and relocated child blocks until the next re-pack
    const size_t room = n_nodes_ + n_nodes_ / 4 + 1024;
    rnodes.reserve(room); rkids.reserve(room); rvals.reserve(n_values_);
    max_depth = 0;
    // iterative pre-order DFS; root children ordered plain-first, `$`-prefixed last (retain.rs:327-331, 345-349)
    using Kids = std::vector<std::pair<u32, u32>>;
    struct Frame { u32 host, dev, next, depth; const Kids* order; };
    Kids root_order = nodes_[0].kids;
    std::stable_partition(root_order.begin(), root_order.end(), [&](const std::pair<u32, u32>& kv) { return !dict_->token_is_dollar(kv.first); });
    std::vector<Frame> stack;
    auto open = [&](u32 host, u32 depth) {
        const HN& h = nodes_[host];
        u32 dev = static_cast<u32>(rnodes.size());
        RNode r{};
        r.first_kid = static_cast<u32>(rkids.size());
        r.nkids = static_cast<u32>(h.kids.size());
        r.val = h.has_val ? h.val : RVAL_NONE;
        r.val_lo = static_cast<u32>(rvals.size());
        r.flags = h.has_val ? 8u : 0u;
        const Kids* order = host == 0 ? &root_order : &h.kids;       // no per-node copy: the host tree is not touched while flattening
        for (const auto& kv : *order) {
            r.pad |= retain_mask_bit(kv.first);
            if (kv.first == TOK_PLUS) r.flags |= RF_LIT_PLUS;
            if (kv.first == TOK_HASH) r.flags |= RF_LIT_HASH | RF_SUB_LIT_HASH;
        }
        rnodes.push_back(r);
        rparent_.push_back(host == 0 ? 0u : nodes_[h.parent].dev); rtoken_.push_back(h.token);
        rcap_.push_back(r.nkids); in_rvals_.push_back(h.has_val ? 1 : 0);
        nodes_[host].dev = dev;
        if (h.has_val) rvals.push_back(h.val);
        rkids.resize(rkids.size() + order->size());
        max_depth = std::max(max_depth, depth);
        stack.push_back(Frame{host, dev, 0, depth, order});
    };
    open(0, 0);
    root_plain_kids = 0;
    for (const auto& kv : root_order) if (!dict_->token_is_dollar(kv.first)) root_plain_kids++;
    root_plain_val_hi = 0;
    while (!stack.empty()) {
        Frame& f = stack.back();
        if (f.next < f.order->size()) {
            u32 j = f.next++;
            if (f.host == 0 && j == root_plain_kids) root_plain_val_hi = static_cast<u32>(rvals.size());
            u32 child_host = (*f.order)[j].second;
            u32 child_dev = static_cast<u32>(rnodes.size());
            RKid& k = rkids[rnodes[f.dev].first_kid + j];
            k.token = (*f.order)[j].first;
            k.child = child_dev;                    // the child's record is copied in below, once its subtree is complete
            open(child_host, f.depth + 1);          // invalidates `f`
        } else {
            RNode& r = rnodes[f.dev];
            r.sub_end = static_cast<u32>(rnodes.size());
            r.val_hi = static_cast<u32>(rvals.size());
            u32 flags = r.flags;
            bool root = f.host == 0;
            u32 parent_dev = 0;
            stack.pop_back();
            if (!stack.empty()) { parent_dev = stack.back().dev; if (flags & RF_SUB_LIT_HASH) rnodes[parent_dev].flags |= RF_SUB_LIT_HASH; }
            if (root && root_plain_kids == nodes_[0].kids.size()) root_plain_val_hi = static_cast<u32>(rvals.size());
        }
    }
    // child entries carry the complete record of the child (flags and value ranges are final only now)
    for (RKid& k : rkids) {
        const RNode& c = rnodes[k.child];
        k.first_kid = c.first_kid; k.nk_flags = c.nkids | (c.flags << 28); k.val = c.val; k.val_lo = c.val_lo; k.val_hi = c.val_hi; k.pad = c.pad;
    }
    // exact-step hash table, load <= 0.25
    size_t cap = 1024;
    while (cap < rkids.size() * 4) cap <<= 1;
    redges.assign_zero(cap);
    const u32 mask = static_cast<u32>(cap - 1);
    // every child entry names its parent implicitly (block of node n): walk nodes, insert their blocks; the first
    // probe slot of the entry 16 ahead is prefetched (the table is far larger than the caches)
    std::vector<u32> parent_of(rkids.size());
    for (u32 n = 0; n < rnodes.size(); ++n)
        for (u32 j = 0; j < rnodes[n].nkids; ++j) parent_of[rnodes[n].first_kid + j] = n;
    for (size_t i = 0; i < rkids.size(); ++i) {
        if (i + 16 < rkids.size()) __builtin_prefetch(&redges[redge_hash(parent_of[i + 16], rkids[i + 16].token) & mask], 1);
        const RKid& k = rkids[i];
        const u32 n = parent_of[i];
        u32 s = redge_hash(n, k.token) & mask;
        while (redges[s].child != 0) s = (s + 1) & mask;
        redges[s] = REdge{n, k.token, k.child, k.first_kid, k.nk_flags, k.val, k.val_lo, k.val_hi};
    }
    // the image is current and packed: ship it whole; from here on set / remove edit it in place
    flat_valid_ = true;
    full = true;
    dirty = true;
    dirty_kids.clear(); dirty_edges.clear(); dirty_vals.clear();
    garbage_kids_ = 0; dead_nodes_ = 0;
    live_edges_ = rkids.size();
    flattens++;
}

}  // namespace gm
