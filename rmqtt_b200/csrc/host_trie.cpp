// Host mirror of the device trie — see host_trie.h.  Mutation semantics follow
// rmqtt/src/trie.rs:99-135 (insert / remove with bottom-up pruning) and the filter validation of
// rmqtt/src/topic.rs:326-363 (Level::from_str, Topic::from_str, Topic::is_valid).
#include "host_trie.h"
#include "host_par.h"

#include <algorithm>
#include <chrono>
#include <queue>
#include <thread>
#include <cstdlib>
#include <cstring>
#include <cstdio>

namespace gm {

namespace {
constexpr u32 NOSLOT = 0xFFFFFFFFu;

inline u32 fnv(const char* s, u32 len) {
    u32 h = FNV_INIT;
    for (u32 i = 0; i < len; ++i) h = fnv_step(h, static_cast<u8>(s[i]));
    return h;
}

// the seven key words of an inline string (<= 27 bytes): bytes, zero padded, length in the last byte
inline void pack_words(const char* s, u32 len, u32 (&w)[7]) {
    u8 b[28] = {0};
    std::memcpy(b, s, len);
    b[27] = static_cast<u8>(len);
    std::memcpy(w, b, 28);
}
inline u32 dict_index_hash(const char* s, u32 len) {
    if (len <= DICT_INLINE_MAX) { u32 w[7]; pack_words(s, len, w); return dict_hash_words(w); }
    return dict_hash_finish(fnv(s, len), len);
}
inline bool dict_slot_equals(const DictSlot& d, const u8* pool, const char* s, u32 len) {
    if (len <= DICT_INLINE_MAX) { u32 w[7]; pack_words(s, len, w); return std::memcmp(&d.w[1], w, 28) == 0; }
    return (d.w[7] >> 24) == 0xFF && d.w[1] == len && d.w[3] == fnv(s, len) && std::memcmp(pool + d.w[2], s, len) == 0;
}
}  // namespace

HostTrie::HostTrie(u32 max_levels) : max_levels_(max_levels) {
    edges.assign_zero(1u << 10);
    dict.assign_zero(1u << 10);
    ranges.assign(1, Range{0, 0});
    cfilter.assign(1u << 10, 0u);
    nodes_.emplace_back();   // root = node 0
    nodes_[0].alive = 1;
    tag_count_.assign(WTAG_COUNT, 0);
    tag_anchors_.assign(WTAG_COUNT, 0);
    // tuning / test knobs: cap on log2(#windows) (0 = one window = plain open addressing) and the smallest window
    if (const char* ev = getenv("GM_EDGE_WINDOWS_LOG2")) { int v = atoi(ev); if (v >= 0 && v <= static_cast<int>(WIN_MAX_LOG2)) nwin_cap_log2_ = static_cast<u32>(v); }
    if (const char* ev = getenv("GM_WIN_MIN_SLOTS_LOG2")) { int v = atoi(ev); if (v >= 3 && v <= 30) win_min_log2_ = static_cast<u32>(v); }
    rehash_edges(edges.size());
}

void HostTrie::reserve(u64 n_filters) {
    // ~2.5 edges and ~0.1 new level strings per filter on IoT-shaped sets.  13 slots per filter keeps the edge
    // table at load ~0.2: on C3, 0.38 -> 0.19 shortens the linear probes of the match kernel; the table of 10 M
    // filters stays a few GB, so HBM capacity (80 GB) is not the constraint.
    u64 per_filter = 13;
    if (const char* ev = getenv("GM_EDGE_SLOTS_PER_FILTER")) { int v = atoi(ev); if (v >= 3 && v <= 64) per_filter = static_cast<u64>(v); }   // tuning knob
    u64 want_e = 1; while (want_e < n_filters * per_filter) want_e <<= 1;
    u64 want_d = 1; while (want_d < n_filters / 2 + 1024) want_d <<= 1;
    want_e = std::min<u64>(want_e, 1ull << 31);
    const bool prof = getenv("GM_BULK_PROFILE") != nullptr;
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = now();
    if (edges.size() < want_e) rehash_edges(static_cast<size_t>(want_e));
    const double t1 = now();
    while (dict.size() < want_d && dict.size() < (1ull << 31)) grow_dict();
    const double t2 = now();
    nodes_.reserve(nodes_.size() + n_filters * 3 + n_filters / 2);
    if (prof) fprintf(stderr, "reserve: edge table %.2f s, dictionary %.2f s, nodes %.2f s\n", t1 - t0, t2 - t1, now() - t2);
}

u32 HostTrie::level0_hash(const char* s, u32 len) {
    u32 l0 = 0;
    while (l0 < len && s[l0] != '/') ++l0;
    return dict_hash_finish(fnv(s, l0), l0);
}

// ------------------------------------------------------------------------------- dictionary
u32 HostTrie::lookup_token(const char* s, u32 len) const {
    if (len == 0) return TOK_BLANK;
    if (len == 1 && s[0] == '+') return TOK_PLUS;
    if (len == 1 && s[0] == '#') return TOK_HASH;
    u32 mask = static_cast<u32>(dict.size() - 1);
    for (u32 i = dict_index_hash(s, len) & mask;; i = (i + 1) & mask) {
        const DictSlot& d = dict[i];
        if (d.w[0] == 0) return TOK_UNKNOWN;
        if (dict_slot_equals(d, pool.data(), s, len)) return d.w[0];
    }
}

u32 HostTrie::intern(const char* s, u32 len, bool create) {
    u32 t = lookup_token(s, len);
    if (t != TOK_UNKNOWN || !create) return t;
    if ((dict_count_ + 1) * 2 > dict.size()) grow_dict();
    u32 mask = static_cast<u32>(dict.size() - 1);
    u32 i = dict_index_hash(s, len) & mask;
    while (dict[i].w[0] != 0) i = (i + 1) & mask;
    DictSlot d{};
    d.w[0] = next_token_++;
    if (len <= DICT_INLINE_MAX) {
        u32 w[7];
        pack_words(s, len, w);
        std::memcpy(&d.w[1], w, 28);
    } else {
        d.w[7] = 0xFFu << 24;
        d.w[1] = len;
        d.w[2] = static_cast<u32>(pool.size());
        d.w[3] = fnv(s, len);
        pool.insert(pool.end(), s, s + len);
        while (pool.size() % 16) pool.push_back(0);
    }
    dict[i] = d;
    dict_count_++;
    if (tok_dollar_.size() <= d.w[0]) tok_dollar_.resize(d.w[0] + 1, 0);
    tok_dollar_[d.w[0]] = (len > 0 && s[0] == '$') ? 1 : 0;
    if (!full_dict) dirty_dict.push_back(i);
    return d.w[0];
}

void HostTrie::grow_dict() {
    ZeroTable<DictSlot> old;
    old.swap(dict);
    dict.assign_zero(old.size() * 2);
    u32 mask = static_cast<u32>(dict.size() - 1);
    for (const DictSlot& d : old) {
        if (d.w[0] == 0) continue;
        u32 h;
        if ((d.w[7] >> 24) == 0xFF) h = dict_hash_finish(d.w[3], d.w[1]);
        else { u32 w[7]; std::memcpy(w, &d.w[1], 28); h = dict_hash_words(w); }
        u32 i = h & mask;
        while (dict[i].w[0] != 0) i = (i + 1) & mask;
        dict[i] = d;
    }
    full_dict = true;
    dirty_dict.clear();
}

// ------------------------------------------------------------------------------- edges
u32 HostTrie::find_edge(u32 parent, u32 token, u32 wtag) const {
    const u32 wm = win_mask();
    for (u32 i = edge_slot0(parent, token, wtag, wm, win_shift(), nwin_mask());; i = edge_next(i, wm)) {
        const EdgeSlot& e = edges[i];
        if (e.child == 0) return NOSLOT;
        if (e.parent == parent && e.token == token) return i;
    }
}

// Re-place every edge into a table of `new_size` slots cut into as many windows as the cap and the minimum
// window size allow.  Tags stay; the effective window is tag & (nwin - 1).
void HostTrie::rehash_edges(size_t new_size) {
    ZeroTable<EdgeSlot> old;
    old.swap(edges);
    edges.assign_zero(new_size);
    u32 bits = 0; while ((size_t(1) << bits) < new_size) ++bits;
    table_log2 = bits;
    nwin_log2 = std::min(nwin_cap_log2_, bits > win_min_log2_ ? bits - win_min_log2_ : 0u);
    win_count_.assign(size_t(1) << nwin_log2, 0);
    const u32 wm = win_mask(), ws = win_shift(), nm = nwin_mask();
    for (const EdgeSlot& e : old) {
        if (e.child == 0) continue;
        const u32 tag = nodes_[e.parent].wtag;
        u32 i = edge_slot0(e.parent, e.token, tag, wm, ws, nm);
        while (edges[i].child != 0) i = edge_next(i, wm);
        edges[i] = e;
        nodes_[e.child].edge_slot = i;
        win_count_[tag & nm]++;
    }
    full_edges = true;
    dirty_edges.clear();
    root_dirty = true;       // the geometry travels with the root record
    for (u32 id = 0; id < nodes_.size(); ++id)      // records name their '+' child by slot: republish them
        if (nodes_[id].plus_child && !nodes_[id].dirty) { nodes_[id].dirty = 1; dirty_nodes_.push_back(id); }
}

// Keeps every window (and so the table) at most half full.  A window that fills while the table as a whole is
// sparse means one subtree outgrew it: double the window size (half as many windows); otherwise double the table
// (same window size, twice as many windows up to the cap).
void HostTrie::make_room(u32 wtag) {
    for (;;) {
        const u64 win_slots = edges.size() >> nwin_log2;
        if ((edge_count_ + 1) * 2 <= edges.size() && (win_count_[wtag & nwin_mask()] + 1) * 2 <= win_slots) return;
        if (getenv("GM_DEBUG_REHASH")) fprintf(stderr, "make_room: tag %u window %u count %llu of %llu slots, edges %llu of %zu, nwin_log2 %u\n", wtag, wtag & nwin_mask(),
                                               (unsigned long long)win_count_[wtag & nwin_mask()], (unsigned long long)win_slots, (unsigned long long)edge_count_, edges.size(), nwin_log2);
        if ((edge_count_ + 1) * 4 > edges.size() || nwin_log2 == 0) rehash_edges(edges.size() * 2);
        else { win_min_log2_ = win_shift() + 2; rehash_edges(edges.size()); }   // x4 per step: at most 4 re-hashes down to one window
    }
}

u32 HostTrie::pick_tag() {
    // tag 0 = the hot window of the top two levels.  Load of a tag = its child edges + a nominal weight per subtree
    // already assigned to it: a new subtree has no edges yet, and a bulk load creates many subtrees back to back
    // (level-synchronously) before any of their children — counting edges alone would give them all the same tag.
    // Exact least-loaded choice while subtrees are few; the better of two hashed candidates once there are many
    // (O(1) per new subtree, still balanced).
    auto load = [&](u32 t) { return tag_count_[t] + 64u * tag_anchors_[t]; };
    u32 best = 1;
    if (anchors_ < 4096) {
        for (u32 t = 2; t < WTAG_COUNT; ++t) if (load(t) < load(best)) best = t;
    } else {
        const u32 h = fmix32(static_cast<u32>(anchors_) * 0x9E3779B1u + 0x7F4A7C15u);
        const u32 a = 1u + (h & 0xFFFFu) % (WTAG_COUNT - 1), b = 1u + (h >> 16) % (WTAG_COUNT - 1);
        best = load(b) < load(a) ? b : a;
    }
    tag_anchors_[best]++;
    anchors_++;
    return best;
}

u32 HostTrie::add_edge(u32 parent, u32 token) {
    const u32 ptag = nodes_[parent].wtag;
    make_room(ptag);
    u32 id = static_cast<u32>(nodes_.size());
    nodes_.emplace_back();
    HNode& n = nodes_.back();
    n.parent = parent;
    n.token = token;
    n.depth = static_cast<uint16_t>(nodes_[parent].depth + 1);
    // where this node's OWN children will live: depth 1 -> hot window 0; depth 2 -> a fresh least-loaded window
    // for the whole subtree; deeper -> inherited
    n.wtag = n.depth <= 1 ? 0 : (n.depth == 2 ? static_cast<u8>(pick_tag()) : static_cast<u8>(ptag));
    const u32 wm = win_mask();
    u32 i = edge_slot0(parent, token, ptag, wm, win_shift(), nwin_mask());
    while (edges[i].child != 0) i = edge_next(i, wm);
    EdgeSlot e{};
    e.parent = parent; e.token = token; e.child = id;
    e.plus = 0; e.hash_ref = 0; e.own_ref = 0; e.mask = static_cast<u32>(n.wtag) << WTAG_SHIFT; e.cnts = 0;
    edges[i] = e;
    n.edge_slot = i;
    edge_count_++;
    tag_count_[ptag]++;
    win_count_[ptag & nwin_mask()]++;
    if (!full_edges) dirty_edges.push_back(i);
    HNode& p = nodes_[parent];
    p.mask |= mask_bit(token);
    if (token != TOK_PLUS && token != TOK_HASH) p.lit_children++;
    if (p.wide) cfilter_insert(parent, token);
    else if (p.lit_children > WIDE_FANOUT) { p.wide = 1; cfilter_rebuild_ = true; }   // its earlier children are back-filled by the rebuild
    if (token == TOK_PLUS) {
        p.plus_child = id;
        plus_count_++;
    } else if (token == TOK_HASH) {
        p.hash_child = id;
    }
    mark(parent);
    return id;
}

// ------------------------------------------------------------------------------- child filter
void HostTrie::cfilter_insert(u32 parent, u32 token) {
    if (cfilter_rebuild_) return;                                   // a rebuild is pending anyway
    if ((cfilter_keys_ + 1) * 16 > cfilter.size() * 32) { cfilter_rebuild_ = true; return; }   // keep >= 16 bits per edge
    u32 w, bits;
    cfilter_pos(parent, token, static_cast<u32>(cfilter.size() - 1), w, bits);
    cfilter[w] |= bits;
    cfilter_keys_++;
    cfilter_dirty = true;
}

void HostTrie::cfilter_rebuild() {
    // every child edge of a wide node; walked over the node array (sequential, one entry per edge) — the edge table itself
    // is mostly empty slots (load 0.2) and several GB at scale.  Big tries: all host threads, bits set with atomic ORs.
    const size_t nn = nodes_.size();
    const unsigned T = nn >= host_par_min(size_t(1) << 18) ? host_threads() : 1u;
    std::vector<u64> cnt(T, 0);
    parallel_chunks(nn, T, [&](unsigned tid, size_t b, size_t e) {
        u64 c = 0;
        for (size_t id = std::max<size_t>(b, 1); id < e; ++id) if (nodes_[nodes_[id].parent].wide) ++c;
        cnt[tid] = c;
    });
    u64 n = 0;
    for (u64 c : cnt) n += c;
    size_t words = 1u << 10;
    while (words * 32 < n * 20) words <<= 1;                        // ~20 bits per edge after a rebuild
    cfilter.assign(words, 0u);
    const u32 mask = static_cast<u32>(words - 1);
    parallel_chunks(nn, T, [&](unsigned, size_t b, size_t e) {
        for (size_t id = std::max<size_t>(b, 1); id < e; ++id) {
            const HNode& c = nodes_[id];
            if (!nodes_[c.parent].wide) continue;
            u32 w, bits;
            cfilter_pos(c.parent, c.token, mask, w, bits);
            if (T > 1) __atomic_fetch_or(&cfilter[w], bits, __ATOMIC_RELAXED); else cfilter[w] |= bits;
        }
    });
    cfilter_keys_ = n;
    cfilter_rebuild_ = false;
    cfilter_dirty = true;
}

// dirty bit 0: the node's record must be re-published; bit 1: its VALUE SET changed (a new reference is needed).
// Only the second kind appends to `values` — a node that merely gained a child edge keeps its published set.
void HostTrie::mark(u32 node) {
    if (!nodes_[node].dirty) dirty_nodes_.push_back(node);
    nodes_[node].dirty |= 1;
}
void HostTrie::mark_vals(u32 node) {
    if (!nodes_[node].dirty) dirty_nodes_.push_back(node);
    nodes_[node].dirty |= 3;
}

// ------------------------------------------------------------------------------- parsing
// Topic::from_str for a *filter*: split on '/', classify every level, validate (topic.rs:326-363,
// :204-216).  Produces tokens; creates dictionary entries when intern_new.
int HostTrie::parse(const char* f, u32 len, bool intern_new, std::vector<u32>& toks) {
    toks.clear();
    u32 start = 0;
    for (;;) {
        u32 end = start;
        bool wild = false;
        while (end < len && f[end] != '/') { wild |= (f[end] == '+' || f[end] == '#'); ++end; }
        u32 l = end - start;
        bool last = end >= len;
        u32 tok;
        if (l == 0) tok = TOK_BLANK;
        else if (l == 1 && f[start] == '+') tok = TOK_PLUS;
        else if (l == 1 && f[start] == '#') { if (!last) return PARSE_INVALID; tok = TOK_HASH; }
        else if (wild) return PARSE_INVALID;
        else {
            if (f[start] == '$' && !toks.empty()) return PARSE_INVALID;   // Metadata only at level 0
            tok = 0xFFFFFFFFu;  // resolved below, after the whole filter validated
        }
        toks.push_back(tok);
        if (toks.size() > max_levels_) return PARSE_TOO_DEEP;
        if (last) break;
        start = end + 1;
    }
    // second pass: dictionary (only now, so an invalid filter never pollutes the dictionary)
    start = 0;
    for (size_t k = 0; k < toks.size(); ++k) {
        u32 end = start;
        while (end < len && f[end] != '/') ++end;
        if (toks[k] == 0xFFFFFFFFu) toks[k] = intern(f + start, end - start, intern_new);
        start = end + 1;
    }
    return PARSE_OK;
}

// ------------------------------------------------------------------------------- mutations
bool HostTrie::add_value(u32 node, u32 value) {
    HNode& n = nodes_[node];
    bool ch = false;
    if (n.nvals == 0) { n.v0 = value; n.nvals = 1; ch = true; }
    else if (n.nvals == 1) {
        if (n.v0 != value) {
            std::vector<u32>& m = multi_[node];
            m = {std::min(n.v0, value), std::max(n.v0, value)};
            n.nvals = 2; ch = true;
        }
    } else {
        std::vector<u32>& m = multi_[node];
        auto it = std::lower_bound(m.begin(), m.end(), value);
        if (it == m.end() || *it != value) { m.insert(it, value); n.nvals++; ch = true; }
    }
    if (ch) {
        values_size_++;
        mark_vals(node);
        if (n.token == TOK_HASH) mark(n.parent);
        // revive pruned ancestors
        for (u32 x = node; x != 0 && !nodes_[x].alive; x = nodes_[x].parent) {
            nodes_[x].alive = 1;
            nodes_[nodes_[x].parent].live_children++;
            live_nodes_++;
        }
    }
    // else: trie.rs:_insert creates the path even when the value was already present; the path exists and is alive
    // in that case by construction (a present value keeps it alive).
    return ch;
}

// Extra trees are children of the global root under a reserved level string that no topic or filter can produce (it
// contains '/', and levels are what is left after splitting on '/').  Nothing can walk into them from tree 0; the kernels
// start a row's walk at its tree's root record (TrieView::tree_slots).
u32 HostTrie::tree_root(u32 tree, bool create) {
    if (tree == 0) return 0;
    if (tree < tree_nodes_.size() && tree_nodes_[tree]) return tree_nodes_[tree];
    if (!create || tree >= MAX_TREES) return 0;
    char name[32];
    const int nl = snprintf(name, sizeof name, "/tree/%u", tree);
    const u32 tok = intern(name, static_cast<u32>(nl), true);
    const u32 slot = find_edge(0, tok, nodes_[0].wtag);
    const u32 id = slot == NOSLOT ? add_edge(0, tok) : edges[slot].child;
    if (tree_nodes_.size() <= tree) tree_nodes_.resize(tree + 1, 0u);
    tree_nodes_[tree] = id;
    tree_of_token_[tok] = tree;
    trees_dirty = true;
    return id;
}

int HostTrie::insert(const char* filter, u32 len, u32 value, bool* changed, u32 tree) {
    if (changed) *changed = false;
    if (tree >= MAX_TREES) return PARSE_INVALID;
    int st = parse(filter, len, true, scratch_toks_);
    if (st != PARSE_OK) return st;
    u32 node = tree_root(tree, true), tag = nodes_[node].wtag;     // the window tag of a node travels in its record (mask word): no lookup in nodes_ per level
    for (u32 tok : scratch_toks_) {
        u32 slot = find_edge(node, tok, tag);
        if (slot == NOSLOT) { node = add_edge(node, tok); tag = nodes_[node].wtag; }
        else { node = edges[slot].child; tag = edges[slot].mask >> WTAG_SHIFT; }
    }
    max_depth = std::max<u32>(max_depth, static_cast<u32>(scratch_toks_.size()));
    const bool ch = add_value(node, value);
    if (changed) *changed = ch;
    return PARSE_OK;
}

// Bulk insert (Raft restore / start-up, rmqtt-cluster-raft/src/router.rs:557-561 re-inserts every filter): the same
// result as n calls of insert(), but walked LEVEL-SYNCHRONOUSLY in groups of 64 filters so that the dependent
// random probes of the multi-GB edge table overlap: pass 1 of a level prefetches every filter's first probe slot,
// pass 2 resolves them in order (creating nodes exactly as the one-by-one path would).
u64 HostTrie::insert_batch(const char* blob, const u32* offsets, const u32* vals, u64 n) {
    if (n >= host_par_min(1u << 16) && host_threads() > 1 && !getenv("GM_BULK_SERIAL")) return insert_batch_parallel(blob, offsets, vals, n, host_threads());
    constexpr u32 G = 64;
    u64 changed = 0;
    const bool prof = getenv("GM_BULK_PROFILE") != nullptr;
    double t_parse = 0, t_walk = 0, t_val = 0;
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    std::vector<u32> toks;                    // tokens of the group, concatenated
    u32 t_off[G + 1], node[G], tag[G];
    u64 idx[G];
    for (u64 base = 0; base < n; base += G) {
        const u32 g = static_cast<u32>(std::min<u64>(G, n - base));
        toks.clear();
        u32 m = 0, deepest = 0;
        t_off[0] = 0;
        double ta = prof ? now() : 0;
        for (u32 j = 0; j < g; ++j) {           // dictionary slots of every level of the group: prefetch before the real parse
            const char* f = blob + offsets[base + j];
            const u32 len = offsets[base + j + 1] - offsets[base + j];
            const u32 dmask = static_cast<u32>(dict.size() - 1);
            for (u32 a = 0; a <= len;) {
                u32 b = a;
                while (b < len && f[b] != '/') ++b;
                if (b > a) __builtin_prefetch(&dict[dict_index_hash(f + a, b - a) & dmask]);
                a = b + 1;
            }
        }
        for (u32 j = 0; j < g; ++j) {
            const u64 i = base + j;
            if (parse(blob + offsets[i], offsets[i + 1] - offsets[i], true, scratch_toks_) != PARSE_OK) continue;   // invalid: skipped like insert()
            toks.insert(toks.end(), scratch_toks_.begin(), scratch_toks_.end());
            idx[m] = i; node[m] = 0; tag[m] = 0;
            t_off[m + 1] = static_cast<u32>(toks.size());
            deepest = std::max<u32>(deepest, static_cast<u32>(scratch_toks_.size()));
            ++m;
        }
        double tb = prof ? now() : 0;
        for (u32 d = 0; d < deepest; ++d) {
            const u32 wm = win_mask(), ws = win_shift(), nm = nwin_mask();
            for (u32 j = 0; j < m; ++j)
                if (t_off[j] + d < t_off[j + 1]) __builtin_prefetch(&edges[edge_slot0(node[j], toks[t_off[j] + d], tag[j], wm, ws, nm)]);
            for (u32 j = 0; j < m; ++j) {
                if (t_off[j] + d >= t_off[j + 1]) continue;
                const u32 tok = toks[t_off[j] + d];
                const u32 slot = find_edge(node[j], tok, tag[j]);
                if (slot == NOSLOT) { node[j] = add_edge(node[j], tok); tag[j] = nodes_[node[j]].wtag; }
                else { node[j] = edges[slot].child; tag[j] = edges[slot].mask >> WTAG_SHIFT; __builtin_prefetch(&nodes_[node[j]]); }   // add_edge below it / add_value will touch it
            }
        }
        max_depth = std::max<u32>(max_depth, deepest);
        double tc = prof ? now() : 0;
        for (u32 j = 0; j < m; ++j) changed += add_value(node[j], vals[idx[j]]) ? 1 : 0;
        if (prof) { const double td = now(); t_parse += tb - ta; t_walk += tc - tb; t_val += td - tc; }
    }
    if (prof) fprintf(stderr, "insert_batch: %llu filters: parse+intern %.2f s, edge walk %.2f s, values %.2f s\n", (unsigned long long)n, t_parse, t_walk, t_val);
    return changed;
}

// ------------------------------------------------------------------------------- parallel bulk insert
// The same trie CONTENT as n calls of insert() (same dictionary numbering too: tokens are assigned in the order of first
// occurrence), built by all host threads.  Node numbers differ from the one-by-one path: they follow the sorted
// (parent, token) order of every level — deterministic, independent of the thread count.
//
//   A  levels -> tokens: every thread validates its share of the filters (Topic::from_str rules, topic.rs:326-363) and
//      collects the level strings the dictionary does not hold in a private set, remembering where each first occurred;
//      the sets are merged in first-occurrence order (serial: ~0.1 string per filter), then every thread resolves its levels.
//   B  one pass per level: (1) every filter looks its edge up (read-only probes of the edge table); the misses are new
//      edges — (2) their keys are sorted and made unique over all threads, (3) node numbers, window tags and room in the
//      table are settled serially, (4) every WINDOW of the table is owned by one thread, which places the new edges of its
//      windows and updates their parents (all children of a node live in one window: no two threads touch the same parent
//      or the same region of the table), (5) the filters that missed look their edge up again.
//   C  values, in filter order (the multi-value sets are a host map).
namespace {
struct LocalStrings {        // level strings one thread met that the dictionary did not hold (open addressing over `ents`)
    struct Ent { const char* s; u32 len, hash; u64 ord; u32 tok; };
    std::vector<Ent> ents;
    std::vector<u32> index;  // hash -> entry + 1
    std::vector<std::vector<u32>> parts;   // entries by partition of the hash space (filled once the set is complete)
    LocalStrings() { index.assign(1u << 12, 0u); }
    static unsigned part_of(u32 hash, unsigned nparts) { return (hash >> 7) % nparts; }
    void partition(unsigned nparts) {
        parts.assign(nparts, {});
        for (u32 k = 0; k < ents.size(); ++k) parts[part_of(ents[k].hash, nparts)].push_back(k);
    }
    u32 add(const char* s, u32 len, u32 h, u64 ord) {
        if ((ents.size() + 1) * 2 > index.size()) {
            std::vector<u32> bigger(index.size() * 2, 0u);
            const size_t m = bigger.size() - 1;
            for (u32 k = 0; k < ents.size(); ++k) { size_t i = ents[k].hash & m; while (bigger[i]) i = (i + 1) & m; bigger[i] = k + 1; }
            index.swap(bigger);
        }
        const size_t m = index.size() - 1;
        for (size_t i = h & m;; i = (i + 1) & m) {
            if (!index[i]) { ents.push_back(Ent{s, len, h, ord, 0u}); index[i] = static_cast<u32>(ents.size()); return static_cast<u32>(ents.size() - 1); }
            const Ent& e = ents[index[i] - 1];
            if (e.hash == h && e.len == len && std::memcmp(e.s, s, len) == 0) return index[i] - 1;   // first occurrence stays: a chunk is walked in order
        }
    }
};
constexpr u32 TOK_LOCAL = 0x80000000u;   // provisional token: index into the thread's LocalStrings
}  // namespace

// Phase A of the bulk paths (also used by the retained tree's bulk load): level strings -> tokens on all threads.
void HostTrie::tokenize_batch(const char* blob, const u32* offsets, u64 n, unsigned T, TokenizedBatch& tb) {
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_begin = now();
    // ---- A0: level offsets (levels of filter i = its '/' count + 1)
    BigVec<u64>& lvl_off = tb.lvl_off;
    lvl_off.assign(n + 1, 0);
    parallel_chunks(n, T, [&](unsigned, size_t b, size_t e) {
        for (size_t i = b; i < e; ++i) {
            const char* f = blob + offsets[i];
            const u32 len = offsets[i + 1] - offsets[i];
            u64 c = 1;
            for (u32 k = 0; k < len; ++k) c += f[k] == '/';
            lvl_off[i + 1] = c;
        }
    });
    for (u64 i = 0; i < n; ++i) lvl_off[i + 1] += lvl_off[i];
    BigVec<u32>& toks = tb.toks;
    BigVec<uint16_t>& depth = tb.depth;
    toks.assign(lvl_off[n], 0u);
    depth.assign(n, 0);                         // 0 = invalid / too deep: skipped like insert()
    // ---- A1: validate + tokens the dictionary already holds
    std::vector<LocalStrings> locals(T);
    std::vector<std::pair<size_t, size_t>> chunk_of(T, {0, 0});
    const bool dict_empty = dict_count_ == 0;
    parallel_chunks(n, T, [&](unsigned tid, size_t b, size_t e) {
        chunk_of[tid] = {b, e};
        LocalStrings L;                          // thread-private while it grows (the objects of `locals` share cache lines)
        for (size_t i = b; i < e; ++i) {
            const char* f = blob + offsets[i];
            const u32 len = offsets[i + 1] - offsets[i];
            u32* out = toks.data() + lvl_off[i];
            // pass 1: shape (an invalid filter never reaches the dictionary)
            bool ok = true;
            u32 nl = 0;
            for (u32 start = 0;;) {
                u32 end = start;
                bool wild = false;
                while (end < len && f[end] != '/') { wild |= (f[end] == '+' || f[end] == '#'); ++end; }
                const u32 l = end - start;
                const bool last = end >= len;
                if (l == 0) out[nl] = TOK_BLANK;
                else if (l == 1 && f[start] == '+') out[nl] = TOK_PLUS;
                else if (l == 1 && f[start] == '#') { if (!last) { ok = false; break; } out[nl] = TOK_HASH; }
                else if (wild) { ok = false; break; }
                else { if (f[start] == '$' && nl) { ok = false; break; } out[nl] = TOK_UNKNOWN; }
                if (++nl > max_levels_) { ok = false; break; }
                if (last) break;
                start = end + 1;
            }
            if (!ok) continue;
            depth[i] = static_cast<uint16_t>(nl);
            // pass 2: literal levels
            u32 k = 0;
            for (u32 start = 0; k < nl; ++k) {
                u32 end = start;
                while (end < len && f[end] != '/') ++end;
                if (out[k] == TOK_UNKNOWN) {
                    const u32 l = end - start;
                    u32 t = dict_empty ? TOK_UNKNOWN : lookup_token(f + start, l);
                    if (t == TOK_UNKNOWN) t = TOK_LOCAL | L.add(f + start, l, dict_index_hash(f + start, l), (static_cast<u64>(i) << 16) | std::min<u32>(k, 65535u));
                    out[k] = t;
                }
                start = end + 1;
            }
        }
        L.partition(T);
        locals[tid] = std::move(L);
    });
    const double t_a1 = now();
    // ---- A2: new level strings enter the dictionary in the order of their first occurrence (what one-by-one inserts do).
    //      The threads' sets overlap (a device name is met by every thread): partition r of the hash space is made unique by
    //      thread r (smallest first occurrence wins); what is left is one entry per new string, interned serially in order.
    {
        struct New { u64 ord; const char* s; u32 len; };
        std::vector<std::vector<New>> uniq(T);
        parallel_threads(T, [&](unsigned r) {
            LocalStrings U;
            for (const LocalStrings& L : locals) {
                if (L.parts.size() != T) continue;        // a thread without a chunk
                for (u32 idx : L.parts[r]) {
                    const auto& e = L.ents[idx];
                    const u32 k = U.add(e.s, e.len, e.hash, e.ord);
                    if (e.ord < U.ents[k].ord) { U.ents[k].ord = e.ord; U.ents[k].s = e.s; }
                }
            }
            std::vector<New> out;
            out.reserve(U.ents.size());
            for (const auto& e : U.ents) out.push_back(New{e.ord, e.s, e.len});
            std::sort(out.begin(), out.end(), [](const New& a, const New& b) { return a.ord < b.ord; });
            uniq[r].swap(out);
        });
        // token of a new string = next_token_ + its rank in first-occurrence order; the strings enter the table on all threads
        // (a slot is claimed by a CAS on its token word: nobody reads the table during this phase, and all strings are distinct)
        std::vector<std::vector<u64>> ords(T);
        parallel_threads(T, [&](unsigned r) { ords[r].reserve(uniq[r].size()); for (const New& x : uniq[r]) ords[r].push_back(x.ord); });
        std::vector<u64> all_ord;
        merge_sorted_unique(ords, T, all_ord);
        const size_t total = all_ord.size();
        if (total) {
            if (static_cast<u64>(next_token_) + total >= TOK_LOCAL) { fprintf(stderr, "gpumqtt: more than 2^31 level strings\n"); std::abort(); }
            while ((dict_count_ + total) * 2 > dict.size()) grow_dict();
            // long strings live in the pool, in token order, each padded to 16 bytes (as intern() lays them out)
            BigVec<u32> plen(total, 0u);
            std::vector<std::vector<u32>> rank(T);
            parallel_threads(T, [&](unsigned r) {
                rank[r].resize(uniq[r].size());
                size_t g = 0;
                for (size_t k = 0; k < uniq[r].size(); ++k) {                      // both sorted by first occurrence
                    while (all_ord[g] != uniq[r][k].ord) ++g;
                    rank[r][k] = static_cast<u32>(g);
                    if (uniq[r][k].len > DICT_INLINE_MAX) plen[g] = (uniq[r][k].len + 15u) & ~15u;
                }
            });
            const size_t pool_base = pool.size();
            u64 run = 0;
            for (size_t g = 0; g < total; ++g) { const u32 l = plen[g]; plen[g] = static_cast<u32>(run); run += l; }
            if (pool_base + run > 0xFFFFFFF0ull) { fprintf(stderr, "gpumqtt: level-string pool exceeds 4 GiB\n"); std::abort(); }
            pool.resize(pool_base + run, 0);
            tok_dollar_.resize(std::max<size_t>(tok_dollar_.size(), static_cast<size_t>(next_token_) + total), 0);
            const u32 dmask = static_cast<u32>(dict.size() - 1);
            const u32 tok0 = next_token_;
            std::vector<std::vector<u32>> t_dirty(T);
            parallel_threads(T, [&](unsigned r) {
                std::vector<u32> dl;
                for (size_t k = 0; k < uniq[r].size(); ++k) {
                    const New& x = uniq[r][k];
                    const u32 tok = tok0 + rank[r][k];
                    DictSlot d{};
                    d.w[0] = tok;
                    if (x.len <= DICT_INLINE_MAX) { u32 w[7]; pack_words(x.s, x.len, w); std::memcpy(&d.w[1], w, 28); }
                    else {
                        const u32 off = static_cast<u32>(pool_base + plen[rank[r][k]]);
                        d.w[7] = 0xFFu << 24; d.w[1] = x.len; d.w[2] = off; d.w[3] = fnv(x.s, x.len);
                        std::memcpy(pool.data() + off, x.s, x.len);
                    }
                    u32 i = dict_index_hash(x.s, x.len) & dmask;
                    for (;; i = (i + 1) & dmask) {
                        u32 expect = 0;
                        if (__atomic_compare_exchange_n(&dict[i].w[0], &expect, tok, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) break;
                    }
                    std::memcpy(&dict[i].w[1], &d.w[1], 28);
                    tok_dollar_[tok] = (x.len > 0 && x.s[0] == '$') ? 1 : 0;
                    if (!full_dict) dl.push_back(i);
                }
                t_dirty[r].swap(dl);
            });
            for (const auto& dl : t_dirty) dirty_dict.insert(dirty_dict.end(), dl.begin(), dl.end());
            dict_count_ += total;
            next_token_ += static_cast<u32>(total);
        }
    }
    const double t_a2 = now();
    // ---- A3: resolve the provisional tokens
    parallel_threads(T, [&](unsigned tid) {
        LocalStrings& L = locals[tid];
        for (auto& e : L.ents) e.tok = lookup_token(e.s, e.len);
        for (size_t i = chunk_of[tid].first; i < chunk_of[tid].second; ++i) {
            u32* out = toks.data() + lvl_off[i];
            for (u32 k = 0; k < depth[i]; ++k) if (out[k] & TOK_LOCAL) out[k] = L.ents[out[k] & ~TOK_LOCAL].tok;
        }
    });
    tb.t_classify = t_a1 - t_begin; tb.t_dictionary = t_a2 - t_a1; tb.t_resolve = now() - t_a2;
}


u64 HostTrie::insert_batch_parallel(const char* blob, const u32* offsets, const u32* vals, u64 n, unsigned T) {
    const bool prof = getenv("GM_BULK_PROFILE") != nullptr;
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_begin = now();
    TokenizedBatch tb;
    tokenize_batch(blob, offsets, n, T, tb);
    const BigVec<u64>& lvl_off = tb.lvl_off;
    const BigVec<u32>& toks = tb.toks;
    const BigVec<uint16_t>& depth = tb.depth;
    const double t_a3 = now();

    // ---- B: nodes, level by level.  Nodes created by this batch (number >= bulk_first) have no edge in the table until the
    //      placement at the end: a look-up below one of them is a miss without a probe.
    const u32 bulk_first = static_cast<u32>(nodes_.size());
    BigVec<u32> cur(n, 0u);
    BigVec<u8> ctag(n, nodes_[0].wtag);
    u32 deepest = 0;
    for (u64 i = 0; i < n; ++i) deepest = std::max<u32>(deepest, depth[i]);
    std::vector<std::vector<std::pair<u64, u32>>> pairs(T);     // per thread: (edge key, filter) of the misses, sorted by key
    std::vector<std::vector<u64>> mkeys(T);                      // ... their distinct keys
    std::vector<std::vector<u32>> mcount(T);                     // ... and how many filters of the thread wait for each
    BigVec<u32> new_weight;                                      // per new node: filters of the batch that run through its edge
    new_weight.reserve(std::min<u64>(toks.size(), n * 3 + 1024));
    double t_find = 0, t_sort = 0, t_serial = 0, t_nodes = 0, t_lsort = 0, t_find0 = 0, t_assign = 0;
    std::vector<u32> revive_parents;           // dead nodes that gained a (live) child
    for (u32 d = 0; d < deepest; ++d) {
        const double tb0 = now();
        // (1) look-ups
        {
            const u32 wm = win_mask(), ws = win_shift(), nm = nwin_mask();
            parallel_chunks(n, T, [&](unsigned tid, size_t b, size_t e) {
                std::vector<std::pair<u64, u32>> pr; std::vector<u64> mk; std::vector<u32> mc;   // thread-private while they grow; capacity of the last level reused
                pr.swap(pairs[tid]); mk.swap(mkeys[tid]); mc.swap(mcount[tid]);
                pr.clear(); mk.clear(); mc.clear();
                constexpr size_t G = 32;
                for (size_t g0 = b; g0 < e; g0 += G) {
                    const size_t g1 = std::min(e, g0 + G);
                    for (size_t i = g0; i < g1; ++i)
                        if (depth[i] > d && cur[i] < bulk_first) __builtin_prefetch(&edges[edge_slot0(cur[i], toks[lvl_off[i] + d], ctag[i], wm, ws, nm)]);
                    for (size_t i = g0; i < g1; ++i) {
                        if (depth[i] <= d) continue;
                        const u32 tok = toks[lvl_off[i] + d];
                        const u32 slot = cur[i] < bulk_first ? find_edge(cur[i], tok, ctag[i]) : NOSLOT;
                        if (slot == NOSLOT) pr.emplace_back((static_cast<u64>(cur[i]) << 32) | tok, static_cast<u32>(i));
                        else { cur[i] = edges[slot].child; ctag[i] = static_cast<u8>(edges[slot].mask >> WTAG_SHIFT); }
                    }
                }
                const double ts0 = tid == 0 ? now() : 0;
                std::sort(pr.begin(), pr.end());
                for (size_t k = 0; k < pr.size(); ++k) { if (k && pr[k].first == pr[k - 1].first) mc.back()++; else { mk.push_back(pr[k].first); mc.push_back(1u); } }
                if (tid == 0) { t_lsort += now() - ts0; t_find0 += ts0 - tb0; }
                pr.swap(pairs[tid]); mk.swap(mkeys[tid]); mc.swap(mcount[tid]);
            });
        }
        const double tb1 = now();
        t_find += tb1 - tb0;
        // (2) new edges of this level: sorted, unique over all threads
        std::vector<u64> ukeys;
        merge_sorted_unique(mkeys, T, ukeys);
        if (ukeys.empty()) continue;                   // every edge of this level existed
        const size_t nu = ukeys.size();
        const double tb2 = now();
        t_sort += tb2 - tb1;
        // (3) node numbers; weights; window tags of new depth-2 subtrees
        const size_t first_new = nodes_.size();
        if (first_new + nu > 0xFFFFFFF0ull) { fprintf(stderr, "gpumqtt: bulk load exceeds 2^32 trie nodes\n"); std::abort(); }
        nodes_.resize(first_new + nu);
        new_weight.resize(first_new - bulk_first + nu, 0u);
        u32* weight = new_weight.data() + (first_new - bulk_first);
        parallel_threads(T, [&](unsigned tid) {
            const auto& mk = mkeys[tid]; const auto& mc = mcount[tid];
            if (mk.empty()) return;
            size_t g = static_cast<size_t>(std::lower_bound(ukeys.begin(), ukeys.end(), mk[0]) - ukeys.begin());
            for (size_t k = 0; k < mk.size(); ++k) { while (ukeys[g] != mk[k]) ++g; __atomic_fetch_add(&weight[g], mc[k], __ATOMIC_RELAXED); }
        });
        if (d == 1) {
            // Window tags of the new depth-2 subtrees.  One-by-one inserts must pick a tag before they know how big a subtree
            // becomes (pick_tag); here every filter of the batch is known: a subtree weighs the filters that run through it, and
            // the heaviest goes first to the least-loaded tag (LPT).  Balanced windows = short probe chains in the match kernel.
            std::vector<u32> order(nu);
            for (size_t g = 0; g < nu; ++g) order[g] = static_cast<u32>(g);
            std::stable_sort(order.begin(), order.end(), [&](u32 a, u32 b) { return weight[a] > weight[b]; });
            using Load = std::pair<u64, u32>;
            std::priority_queue<Load, std::vector<Load>, std::greater<Load>> heap;
            for (u32 t = 1; t < WTAG_COUNT; ++t) heap.push(Load{tag_count_[t] + 64u * tag_anchors_[t], t});
            for (u32 g : order) {
                Load l = heap.top(); heap.pop();
                nodes_[first_new + g].wtag = static_cast<u8>(l.second);
                tag_anchors_[l.second]++; anchors_++;
                l.first += 64u + 3ull * weight[g];           // ~3 edges per filter below depth 2 on IoT-shaped sets; what matters is the proportion
                heap.push(l);
            }
        }
        const double tb3 = now();
        t_serial += tb3 - tb2;
        // (4) the new nodes and what they change in their parents.  The keys are sorted by parent: a thread takes a run of whole
        //     parents, so nothing here is shared between threads.
        {
            std::vector<std::vector<u32>> t_dirty(T), t_revive(T);
            std::vector<u64> t_plus(T, 0);
            std::vector<u8> t_cf(T, 0);
            const u32 child_depth = d + 1;
            parallel_chunks(nu, T, [&](unsigned tid, size_t b, size_t e) {
                auto parent_of = [&](size_t g) { return static_cast<u32>(ukeys[g] >> 32); };
                while (b > 0 && b < nu && parent_of(b) == parent_of(b - 1)) ++b;       // the run of a parent belongs to the chunk it starts in
                while (e > 0 && e < nu && parent_of(e) == parent_of(e - 1)) ++e;
                std::vector<u32> dl, rv; u64 l_plus = 0; u8 l_cf = 0;
                for (size_t g = b; g < e; ++g) {
                    const u32 parent = parent_of(g), token = static_cast<u32>(ukeys[g]);
                    const u32 id = static_cast<u32>(first_new + g);
                    HNode& pn = nodes_[parent];
                    HNode& c = nodes_[id];
                    c.parent = parent; c.token = token; c.depth = static_cast<uint16_t>(child_depth);
                    if (child_depth <= 1) c.wtag = 0; else if (child_depth != 2) c.wtag = pn.wtag;   // depth 2: picked in (3)
                    c.edge_slot = NOSLOT;                  // placed at the end
                    pn.mask |= mask_bit(token);
                    if (token != TOK_PLUS && token != TOK_HASH) pn.lit_children++;
                    if (pn.wide) l_cf = 1;
                    else if (pn.lit_children > WIDE_FANOUT) { pn.wide = 1; l_cf = 1; }
                    if (token == TOK_PLUS) { pn.plus_child = id; l_plus++; }
                    else if (token == TOK_HASH) pn.hash_child = id;
                    if (!pn.dirty) dl.push_back(parent);
                    pn.dirty |= 1;
                    // a bulk-created node always ends up alive (a value is stored at or below it): born alive, counted by its parent;
                    // a DEAD parent (pruned earlier, trie.rs:126-128) is revived after the join
                    c.alive = 1;
                    pn.live_children++;
                    if (!pn.alive) rv.push_back(parent);
                }
                t_revive[tid].swap(rv); t_dirty[tid].swap(dl); t_plus[tid] = l_plus; t_cf[tid] = l_cf;
            });
            for (unsigned t = 0; t < T; ++t) {
                dirty_nodes_.insert(dirty_nodes_.end(), t_dirty[t].begin(), t_dirty[t].end());
                revive_parents.insert(revive_parents.end(), t_revive[t].begin(), t_revive[t].end());
                plus_count_ += t_plus[t];
                if (t_cf[t]) cfilter_rebuild_ = true;     // the child filter is rebuilt from the nodes by the next sync()
            }
            live_nodes_ += nu;
        }
        const double tb4 = now();
        t_nodes += tb4 - tb3;
        // (5) the filters that missed step onto their new node: their sorted (key, filter) pairs against the sorted level
        parallel_threads(T, [&](unsigned tid) {
            const auto& pr = pairs[tid];
            if (pr.empty()) return;
            size_t g = static_cast<size_t>(std::lower_bound(ukeys.begin(), ukeys.end(), pr[0].first) - ukeys.begin());
            for (size_t k = 0; k < pr.size(); ++k) {
                while (ukeys[g] != pr[k].first) ++g;
                const u32 id = static_cast<u32>(first_new + g);
                cur[pr[k].second] = id; ctag[pr[k].second] = nodes_[id].wtag;
            }
        });
        t_assign += now() - tb4;
    }
    // ---- placement of the new edges.  Linear probing gives the home slot to whoever comes first: one-by-one inserts place an
    //      edge when its first filter arrives, so the edges many filters share sit at home and the rare ones are displaced —
    //      and the edges many filters share are the ones PUBLISH topics walk most.  Same rule here, exactly: every window's new
    //      edges go in by descending weight (filters of the batch running through the edge).  Every window belongs to one thread.
    const double t_p0 = now();
    const size_t NB = nodes_.size() - bulk_first;
    if (NB) {
        BigVec<u8> own(NB);
        for (;;) {                                           // room for all of them (more / wider windows, or a bigger table)
            const u32 nm = nwin_mask();
            std::vector<std::vector<u64>> hist(T, std::vector<u64>(size_t(nm) + 1, 0));
            parallel_chunks(NB, T, [&](unsigned tid, size_t b, size_t e) {
                std::vector<u64>& h = hist[tid];
                for (size_t k = b; k < e; ++k) { const u32 w = nodes_[nodes_[bulk_first + k].parent].wtag & nm; own[k] = static_cast<u8>(w); h[w]++; }
            });
            std::vector<u64> add_w(size_t(nm) + 1, 0);
            for (const auto& h : hist) for (size_t w = 0; w <= nm; ++w) add_w[w] += h[w];
            const u64 win_slots = edges.size() >> nwin_log2;
            bool fits = (edge_count_ + NB) * 2 <= edges.size();
            for (size_t w = 0; fits && w <= nm; ++w) fits = (win_count_[w] + add_w[w]) * 2 <= win_slots;
            if (fits) break;
            if ((edge_count_ + NB) * 4 > edges.size() || nwin_log2 == 0) rehash_edges(edges.size() * 2);
            else { win_min_log2_ = win_shift() + 2; rehash_edges(edges.size()); }
        }
        const u32 wm = win_mask(), ws = win_shift(), nm = nwin_mask();
        std::vector<std::vector<u64>> t_tag(T), t_win(T);
        parallel_threads(T, [&](unsigned tid) {
            std::vector<u64> mine;                           // (~weight, node) of this thread's windows: ascending = heaviest first, ties by node number
            for (size_t k = 0; k < NB; ++k) if (own[k] % T == tid) mine.push_back((static_cast<u64>(~new_weight[k]) << 32) | static_cast<u32>(bulk_first + k));
            std::sort(mine.begin(), mine.end());
            std::vector<u64> l_tag(WTAG_COUNT, 0), l_win(size_t(nm) + 1, 0);   // private until the join (neighbouring counters share cache lines)
            for (size_t q = 0; q < mine.size(); ++q) {
                if (q + 8 < mine.size()) {
                    const HNode& c8 = nodes_[static_cast<u32>(mine[q + 8])];
                    __builtin_prefetch(&edges[edge_slot0(c8.parent, c8.token, nodes_[c8.parent].wtag, wm, ws, nm)], 1);
                }
                const u32 id = static_cast<u32>(mine[q]);
                HNode& c = nodes_[id];
                const u32 ptag = nodes_[c.parent].wtag;
                u32 i = edge_slot0(c.parent, c.token, ptag, wm, ws, nm);
                while (edges[i].child != 0) i = edge_next(i, wm);
                EdgeSlot es{};
                es.parent = c.parent; es.token = c.token; es.child = id;
                es.plus = 0; es.hash_ref = 0; es.own_ref = 0; es.mask = static_cast<u32>(c.wtag) << WTAG_SHIFT; es.cnts = 0;
                edges[i] = es;
                c.edge_slot = i;
                l_tag[ptag]++; l_win[ptag & nm]++;
            }
            t_tag[tid].swap(l_tag); t_win[tid].swap(l_win);
        });
        for (unsigned t = 0; t < T; ++t) {
            for (size_t k = 0; k < t_tag[t].size(); ++k) tag_count_[k] += t_tag[t][k];
            for (size_t k = 0; k < t_win[t].size(); ++k) win_count_[k] += t_win[t][k];
        }
        edge_count_ += NB;
        full_edges = true; dirty_edges.clear();              // the placed slots were not listed one by one: the next flush ships the table
    }
    const double t_place = now() - t_p0;
    max_depth = std::max<u32>(max_depth, deepest);
    // ---- C: values.  A node belongs to one thread (blocks of 64 node numbers): it applies the node's values in filter order;
    //      what reaches beyond the node — the host map of multi-value sets, the parent of a '#' node, dead ancestors to
    //      revive — is collected per thread and settled after the join.
    const double t_c = now();
    u64 changed = 0;
    {
        using Multi = std::unordered_map<u32, std::vector<u32>>;
        std::vector<Multi> t_multi(T);
        std::vector<std::vector<u32>> t_dirty(T), t_hashpar(T), t_revive(T);
        std::vector<u64> t_changed(T, 0);
        parallel_threads(T, [&](unsigned tid) {
            Multi lm; std::vector<u32> dl, hp, rv; u64 ch = 0;
            for (u64 i = 0; i < n; ++i) {
                if (!depth[i]) continue;
                const u32 node = cur[i];
                if ((node >> 6) % T != tid) continue;
                HNode& nd = nodes_[node];
                const u32 value = vals[i];
                bool c = false;
                if (nd.nvals == 0) { nd.v0 = value; nd.nvals = 1; c = true; }
                else {
                    std::vector<u32>* m = nullptr;
                    if (nd.nvals >= 2) { auto it = lm.find(node); m = it != lm.end() ? &it->second : &multi_.find(node)->second; }   // an older set lives in the shared map: found, never inserted, by its only writer
                    if (nd.nvals == 1) {
                        if (nd.v0 != value) { lm[node] = {std::min(nd.v0, value), std::max(nd.v0, value)}; nd.nvals = 2; c = true; }
                    } else {
                        auto it = std::lower_bound(m->begin(), m->end(), value);
                        if (it == m->end() || *it != value) { m->insert(it, value); nd.nvals++; c = true; }
                    }
                }
                if (!c) continue;
                ++ch;
                if (!nd.dirty) dl.push_back(node);
                nd.dirty |= 3;
                if (nd.token == TOK_HASH) hp.push_back(nd.parent);
                if (!nd.alive) rv.push_back(node);
            }
            t_multi[tid].swap(lm); t_dirty[tid].swap(dl); t_hashpar[tid].swap(hp); t_revive[tid].swap(rv); t_changed[tid] = ch;
        });
        for (unsigned t = 0; t < T; ++t) {
            changed += t_changed[t];
            multi_.merge(t_multi[t]);
            dirty_nodes_.insert(dirty_nodes_.end(), t_dirty[t].begin(), t_dirty[t].end());
            for (u32 p : t_hashpar[t]) mark(p);
            for (u32 x : t_revive[t])
                for (; x != 0 && !nodes_[x].alive; x = nodes_[x].parent) { nodes_[x].alive = 1; nodes_[nodes_[x].parent].live_children++; live_nodes_++; }
        }
        for (u32 x : revive_parents)
            for (; x != 0 && !nodes_[x].alive; x = nodes_[x].parent) { nodes_[x].alive = 1; nodes_[nodes_[x].parent].live_children++; live_nodes_++; }
        values_size_ += changed;
    }
    if (prof)
        fprintf(stderr, "insert_batch (%u threads): %llu filters: tokens %.2f s (classify %.2f, dictionary %.2f, resolve %.2f), edges %.2f s (look-ups %.2f [thread 0: probes %.2f, local sort %.2f], merge %.2f, numbers + tags %.2f, nodes %.2f, step %.2f, placement %.2f), values %.2f s\n",
                T, (unsigned long long)n, t_a3 - t_begin, tb.t_classify, tb.t_dictionary, tb.t_resolve, t_c - t_a3, t_find, t_find0, t_lsort, t_sort, t_serial, t_nodes, t_assign, t_place, now() - t_c);
    return changed;
}

int HostTrie::remove(const char* filter, u32 len, u32 value, bool* changed, u32 tree) {
    if (changed) *changed = false;
    int st = parse(filter, len, false, scratch_toks_);
    if (st != PARSE_OK) return st;
    u32 node = tree_root(tree, false);
    if (tree && !node) return PARSE_OK;              // no such tree: nothing to remove
    u32 tag = nodes_[node].wtag;
    for (u32 tok : scratch_toks_) {
        if (tok == TOK_UNKNOWN) return PARSE_OK;
        u32 slot = find_edge(node, tok, tag);
        if (slot == NOSLOT) return PARSE_OK;
        node = edges[slot].child;
        tag = edges[slot].mask >> WTAG_SHIFT;
        if (!nodes_[node].alive) return PARSE_OK;      // pruned in the reference: branches.get_mut -> None
    }
    HNode& n = nodes_[node];
    bool ch = false;
    if (n.nvals == 1) { if (n.v0 == value) { n.nvals = 0; ch = true; } }
    else if (n.nvals > 1) {
        std::vector<u32>& m = multi_[node];
        auto it = std::lower_bound(m.begin(), m.end(), value);
        if (it != m.end() && *it == value) {
            m.erase(it); n.nvals--; ch = true;
            if (n.nvals == 1) { n.v0 = m[0]; multi_.erase(node); }
        }
    }
    if (ch) {
        values_size_--;
        mark_vals(node);
        if (n.token == TOK_HASH) mark(n.parent);
    }
    // bottom-up pruning (trie.rs:126-128): a node with no values and no children disappears
    for (u32 x = node; x != 0; x = nodes_[x].parent) {
        HNode& c = nodes_[x];
        if (!(c.alive && c.nvals == 0 && c.live_children == 0)) break;
        c.alive = 0;
        nodes_[c.parent].live_children--;
        live_nodes_--;
    }
    if (changed) *changed = ch;
    return PARSE_OK;
}

// ------------------------------------------------------------------------------- publishing
void HostTrie::make_ref(u32 node) {
    HNode& n = nodes_[node];
    if (n.cnt16 >= 2) garbage_values += (n.cnt16 == CNT_BIG) ? ranges[n.ref].cnt : n.cnt16;   // old copy becomes garbage
    if (n.nvals == 0) { n.ref = 0; n.cnt16 = 0; return; }
    if (n.nvals == 1) { n.ref = n.v0; n.cnt16 = 1; return; }
    const std::vector<u32>& m = multi_[node];
    u32 off = static_cast<u32>(values.size());
    values.append(m.begin(), m.end());
    if (n.nvals < CNT_BIG) { n.ref = off; n.cnt16 = n.nvals; return; }
    n.ref = static_cast<u32>(ranges.size());
    n.cnt16 = CNT_BIG;
    ranges.push_back(Range{off, n.nvals});
}

void HostTrie::write_record(u32 node) {
    const HNode& n = nodes_[node];
    const u32 plus_idx = n.plus_child ? nodes_[n.plus_child].edge_slot + 1u : 0u;   // direct slot of the '+' child
    u32 hash_ref = n.hash_child ? nodes_[n.hash_child].ref : 0;
    u32 hash_cnt = n.hash_child ? nodes_[n.hash_child].cnt16 : 0;
    const u32 mask = (n.mask & MASK_BLOOM) | (n.wide ? MASK_WIDE_FLAG : 0u) | (static_cast<u32>(n.wtag) << WTAG_SHIFT);
    if (node == 0) {
        root_plus = plus_idx; root_hash_ref = hash_ref; root_hash_cnt = hash_cnt; root_mask = mask;
        root_dirty = true;
        return;
    }
    EdgeSlot& e = edges[n.edge_slot];
    e.plus = plus_idx; e.hash_ref = hash_ref; e.own_ref = n.ref; e.mask = mask; e.cnts = hash_cnt | (n.cnt16 << 16);
    if (!full_edges) dirty_edges.push_back(n.edge_slot);
}

void HostTrie::compact(const std::vector<u32>* keep, std::vector<u32>* remap) {
    // token -> level string, from the dictionary slots
    std::vector<std::string> tok_str(next_token_);
    for (const DictSlot& d : dict) {
        if (d.w[0] == 0) continue;
        if ((d.w[7] >> 24) == 0xFF) tok_str[d.w[0]].assign(reinterpret_cast<const char*>(pool.data() + d.w[2]), d.w[1]);
        else { const char* b = reinterpret_cast<const char*>(&d.w[1]); tok_str[d.w[0]].assign(b, d.w[7] >> 24); }
    }
    tok_str[TOK_PLUS] = "+"; tok_str[TOK_HASH] = "#"; tok_str[TOK_BLANK] = "";
    HostTrie fresh(max_levels_);
    fresh.reserve(values_size_);
    std::vector<u32> path;
    std::string f;
    for (u32 id = 1; id < nodes_.size(); ++id) {
        const HNode& n = nodes_[id];
        if (n.nvals == 0) continue;
        path.clear();
        for (u32 x = id; x != 0; x = nodes_[x].parent) path.push_back(nodes_[x].token);
        u32 tree = 0;
        auto tt = tree_of_token_.find(path.back());
        if (tt != tree_of_token_.end()) { tree = tt->second; path.pop_back(); }      // the reserved root level of an extra tree
        if (path.empty()) continue;
        f.clear();
        for (size_t k = path.size(); k-- > 0;) { f += tok_str[path[k]]; if (k) f += '/'; }
        bool ch;
        if (n.nvals == 1) fresh.insert(f.data(), static_cast<u32>(f.size()), n.v0, &ch, tree);
        else for (u32 v : multi_[id]) fresh.insert(f.data(), static_cast<u32>(f.size()), v, &ch, tree);
    }
    if (remap) remap->assign(next_token_, 0u);
    if (keep)
        for (u32 old : *keep) {
            if (old < TOK_FIRST || old >= tok_str.size()) continue;
            const u32 neu = fresh.intern(tok_str[old].data(), static_cast<u32>(tok_str[old].size()), true);
            if (remap) (*remap)[old] = neu;
        }
    fresh.values_epoch = values_epoch + 1;           // `values` was rebuilt: descriptors of an earlier epoch are stale (gm_values)
    *this = std::move(fresh);
}

// Drops the garbage copies of replaced value sets: `values` / `ranges` are rebuilt from the live multi-value sets
// (every such node gets a fresh reference and re-publishes its record).  O(multi-value nodes), not O(filters).
void HostTrie::compact_values() {
    values.clear();
    ranges.assign(1, Range{0, 0});
    garbage_values = 0;
    values_epoch++;
    for (auto& kv : multi_) {
        HNode& n = nodes_[kv.first];
        n.ref = 0; n.cnt16 = 0;                       // the old copy is gone: nothing to count as garbage
        mark_vals(kv.first);
        if (n.token == TOK_HASH) mark(n.parent);
    }
}

bool HostTrie::sync() {
    // value words this flush appends; replaced copies become garbage.  Auto-compaction keeps both bounded: churn on
    // one popular filter would otherwise grow `values` without limit and finally wrap the 32-bit references.
    auto pending_words = [&]() {
        const unsigned TT = dirty_nodes_.size() >= host_par_min(size_t(1) << 18) ? host_threads() : 1u;
        std::vector<u64> part(TT, 0);
        parallel_chunks(dirty_nodes_.size(), TT, [&](unsigned tid, size_t b, size_t e) {
            u64 w = 0;
            for (size_t k = b; k < e; ++k) { const HNode& n = nodes_[dirty_nodes_[k]]; if ((n.dirty & 2) && n.nvals >= 2) w += n.nvals; }
            part[tid] = w;
        });
        u64 w = 0;
        for (u64 x : part) w += x;
        return w;
    };
    u64 add_words = pending_words();
    const u64 live_words = values.size() - std::min<u64>(garbage_values, values.size());
    if (garbage_values > live_words + 65536 || values.size() + add_words > 0xFFFFFFF0ull) {
        compact_values();
        add_words = pending_words();
        if (add_words > 0xFFFFFFF0ull) return false;   // more than 2^32 value words live: references would wrap
    }
    const bool prof = getenv("GM_BULK_PROFILE") != nullptr;
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = prof ? now() : 0;
    const unsigned T = dirty_nodes_.size() >= host_par_min(size_t(1) << 18) || nodes_.size() >= host_par_min(size_t(1) << 20) ? host_threads() : 1u;
    if (cfilter_rebuild_) {
        // nodes that just became wide must republish their record (flag)
        std::vector<std::vector<u32>> found(T);
        parallel_chunks(nodes_.size(), T, [&](unsigned tid, size_t b, size_t e) {
            std::vector<u32> f;
            for (size_t id = b; id < e; ++id) if (nodes_[id].wide && !nodes_[id].dirty) { nodes_[id].dirty = 1; f.push_back(static_cast<u32>(id)); }
            found[tid].swap(f);
        });
        for (const auto& f : found) dirty_nodes_.insert(dirty_nodes_.end(), f.begin(), f.end());
        cfilter_rebuild();
    }
    // pass 1: value-set references (a '#' node's parent reads the child's fresh ref in pass 2).  Sets with more than
    // one value are appended to `values`; they are appended grouped by (window, depth-2 subtree) so that the sets
    // one tile of the match kernel expands (same level0/level1 subtree) are neighbours in `values` as well.
    const double t1 = prof ? now() : 0;
    std::vector<std::pair<u64, u32>> multi;
    {
        std::vector<std::vector<std::pair<u64, u32>>> t_multi(T);
        std::vector<u64> t_garbage(T, 0);
        parallel_chunks(dirty_nodes_.size(), T, [&](unsigned tid, size_t b, size_t e) {
            std::vector<std::pair<u64, u32>> lm; u64 garbage = 0;
            for (size_t k = b; k < e; ++k) {
                const u32 id = dirty_nodes_[k];
                HNode& n = nodes_[id];
                if (!(n.dirty & 2)) continue;             // record-only change: the published set stays
                if (n.nvals < 2) {                        // make_ref without the shared counters
                    if (n.cnt16 >= 2) garbage += (n.cnt16 == CNT_BIG) ? ranges[n.ref].cnt : n.cnt16;
                    if (n.nvals == 0) { n.ref = 0; n.cnt16 = 0; } else { n.ref = n.v0; n.cnt16 = 1; }
                    continue;
                }
                u32 a = id;
                while (nodes_[a].depth > 2) a = nodes_[a].parent;
                const u32 tag = id == 0 ? 0u : nodes_[nodes_[id].parent].wtag;
                lm.emplace_back((static_cast<u64>(tag) << 32) | a, id);
            }
            t_multi[tid].swap(lm); t_garbage[tid] = garbage;
        });
        for (unsigned t = 0; t < T; ++t) { multi.insert(multi.end(), t_multi[t].begin(), t_multi[t].end()); garbage_values += t_garbage[t]; }
    }
    std::sort(multi.begin(), multi.end());
    for (const auto& m : multi) make_ref(m.second);
    // pass 2: records.  Every node writes its OWN slot (the root: the root record) from refs that pass 1 has settled, so after a
    // bulk load / re-hash (the whole table ships anyway: no per-slot dirty list to append to) the millions of random
    // slot writes are spread over the host cores.
    const double t2 = prof ? now() : 0;
    const size_t nd = dirty_nodes_.size();
    auto write_range = [&](size_t b, size_t e) {
        for (size_t i = b; i < e; ++i) {
            if (i + 16 < e) __builtin_prefetch(&edges[nodes_[dirty_nodes_[i + 16]].edge_slot], 1);   // records land in random slots
            const u32 id = dirty_nodes_[i];
            write_record(id);
            nodes_[id].dirty = 0;
        }
    };
    const unsigned hw = host_threads();
    if (full_edges && nd >= host_par_min(size_t(1) << 18) && hw > 1 && !getenv("GM_SYNC_SERIAL")) {
        size_t root_at = nd;                              // the root record is shared state (root_*): its node is written by this thread
        for (size_t i = 0; i < nd; ++i) if (dirty_nodes_[i] == 0) { root_at = i; break; }
        if (root_at != nd) std::swap(dirty_nodes_[root_at], dirty_nodes_[nd - 1]);
        const size_t npar = root_at != nd ? nd - 1 : nd;
        std::vector<std::thread> th;
        const size_t chunk = (npar + hw - 1) / hw;
        for (unsigned t = 0; t < hw; ++t) {
            const size_t b = std::min(npar, t * chunk), e = std::min(npar, b + chunk);
            if (b < e) th.emplace_back(write_range, b, e);
        }
        for (auto& t : th) t.join();
        write_range(npar, nd);
    } else write_range(0, nd);
    if (prof && nd > 100000) fprintf(stderr, "sync: %zu dirty nodes: child filter %.2f s, value refs %.2f s, records %.2f s\n", nd, t1 - t0, t2 - t1, now() - t2);
    dirty_nodes_.clear();
    if (tree_nodes_.size() > 1) {                     // root records of the extra trees: their slots move with every re-hash
        std::vector<u32> ts(tree_nodes_.size(), 0xFFFFFFFFu);
        for (size_t k = 1; k < tree_nodes_.size(); ++k) if (tree_nodes_[k]) ts[k] = nodes_[tree_nodes_[k]].edge_slot;
        if (ts != tree_slots) { tree_slots.swap(ts); trees_dirty = true; }
    }
    return true;
}

}  // namespace gm
