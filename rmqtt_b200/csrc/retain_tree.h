// Host mirror + device layout of the retained-message tree (rmqtt/src/retain.rs:202-257).
//
// The tree is keyed by CONCRETE topics (one optional value per node); queries are topic FILTERS:
// '+' = every child, '#' = the whole subtree (retain.rs:298-367).  Device layout (built by `flatten`, then kept up to
// date IN PLACE by set / remove — see "incremental updates" below — and shipped by the engine's flush):
//
//   rnodes : nodes in DFS PRE-ORDER, so the subtree of node n is the index range [n, sub_end(n)) and the
//            values below a node are ONE contiguous range of `rvals` -> a '#' match is a range copy
//   rkids  : per node, its children as a contiguous block of 32-byte entries {token, child, child's record}
//            -> a '+' match is a coalesced scan of one block and yields complete work items
//   redges : open-addressing hash (parent, token) -> child + the child's record for the exact-level steps
//   rvals  : the values of all valued nodes, in pre-order
//
// Incremental updates.  After a flatten the arrays are a packed pre-order image.  A later set / remove edits them
// in place and records which 32-byte entries / words changed (the flush ships only those):
//   * value replaced on a node        -> its record (2 copies: parent's child block, hash slot) + its word in rvals
//   * node gains / loses its value    -> its record; the '#' ranges of the node and of all its ancestors no longer
//                                        describe the subtree, so they get RF_SUB_LIT_HASH ("walk, do not range-copy")
//   * new nodes below an existing one -> appended to rnodes; the parent's child block moves to the end of rkids with
//                                        doubled capacity when it is full (the old block becomes garbage); new
//                                        hash slots; ancestors flagged as above
//   * pruned nodes (retain.rs:247-249) stay behind as dead leaves (no value, no children: they cannot produce a
//     hit) and are revived when the same path is set again
// Anything involving a literal '+' / '#' level (they shadow wildcard expansion), a hash table more than half full,
// or too much garbage falls back to a full flatten at the next flush.
#pragma once
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "host_trie.h"
#include "layout.h"

namespace gm {

constexpr u32 RVAL_NONE = 0xFFFFFFFFu;
constexpr u32 RF_LIT_PLUS = 1u;       // node has a child whose level is literally "+"  (shadows '+' expansion, retain.rs:313)
constexpr u32 RF_LIT_HASH = 2u;       // node has a child whose level is literally "#"
constexpr u32 RF_SUB_LIT_HASH = 4u;   // some node in this subtree (self included) has a literal "#" child:
                                      // the '#' recursion is shadowed somewhere below -> no range shortcut

struct alignas(32) RNode {
    u32 first_kid, nkids;
    u32 val;              // RVAL_NONE = no value
    u32 val_lo, val_hi;   // rvals[val_lo .. val_hi) = values of the subtree [n, sub_end) (own value first)
    u32 flags;
    u32 sub_end;
    u32 pad;              // Bloom mask over the tokens of this node's children (retain_mask_bit); stale bits after removals are harmless
};
// A node's record as the walk needs it: {first_kid, nk_flags, val, val_lo, val_hi} where nk_flags = #kids (28 bits) |
// flags << 28 (RF_* and 8 = has value).  It travels WITH the reference to the node — inside the parent's child
// block entry and inside the (parent, token) hash slot — so visiting a node costs no extra memory access.
constexpr u32 RNK_MASK = 0x0FFFFFFFu;
struct alignas(32) RKid { u32 token, child, first_kid, nk_flags, val, val_lo, val_hi, pad; };   // pad = the child's child-token mask
struct alignas(32) REdge { u32 parent, token, child, first_kid, nk_flags, val, val_lo, val_hi; };   // child == 0: empty (root is node 0)

struct RetainView {
    const RKid* kids;
    const REdge* edges;
    const u32* vals;
    u32 edge_mask;
    u32 root_first_kid, root_nk_flags;
    u32 root_plain_kids;     // root children whose level does not start with '$' (ordered first)
    u32 root_plain_val_hi;   // rvals[0 .. root_plain_val_hi) = values below those children
    u32 max_depth;
    u32 n_kids;              // entries in `kids` (child blocks are laid out in tree pre-order: position in `kids` = position in the tree)
};

// one of 32 bits for a child token: the Bloom mask over a node's children kept in RNode::pad / RKid::pad
GM_HD u32 retain_mask_bit(u32 token) { return 1u << ((token * 0x9E3779B1u) >> 27); }
GM_HD u32 redge_hash(u32 parent, u32 token) { return fmix32(parent * 0x85EBCA77u + (token ^ 0x2545F491u) * 0x9E3779B1u); }

class RetainTreeHost {
  public:
    explicit RetainTreeHost(HostTrie* dict) : dict_(dict) { nodes_.emplace_back(); }

    // RetainTree::insert (retain.rs:221-234): value.replace(v).  Returns ParseStatus or SET_CONFLICT; *had_old / *old as
    // remove.  = set_ttl without a deadline: clears the handle's deadline.
    int set(const char* topic, u32 len, u32 value, bool* had_old, u32* old) { return set_ttl(topic, len, value, 0, had_old, old); }
    // RetainTree::remove (retain.rs:237-257) with bottom-up pruning; clears the deadline of the handle it removes.
    int remove(const char* topic, u32 len, bool* had_old, u32* old);

    // ---- deadlines (RetainStorage::set_with_timeout / remove_expired_messages, retain.rs:118-149) ----
    // A deadline is in ms since the Unix epoch (0 = none) and belongs to a handle; a handle that carries one is stored under
    // one topic only, whose bytes are kept for the sweep.  A value replaced or removed loses its deadline.  `dl` is the
    // handle-indexed table the lookup reads (~0 = none); the flush ships it whole when it grew, else its dirty words.
    static constexpr int SET_CONFLICT = 16;            // status: the handle carries a deadline under another topic (nothing changed)
    static constexpr int SET_HANDLE_RANGE = 17;        // status: a deadline for a handle >= DL_MAX_HANDLE (nothing changed)
    static constexpr u32 DL_MAX_HANDLE = 1u << 28;     // the table takes 8 bytes per handle up to the largest one with a deadline
    static constexpr u64 DL_NONE = ~0ull;
    int set_ttl(const char* topic, u32 len, u32 value, u64 deadline, bool* had_old, u32* old);
    // whether n sets with these deadlines (nullptr: none) would store a handle with a deadline under a second topic
    // (SET_CONFLICT / SET_HANDLE_RANGE) — checked before a batch changes anything; PARSE_OK otherwise
    int check_batch(const char* blob, const u32* offsets, const u32* values, const u64* deadlines, u64 n) const;
    // set_batch, then the deadlines of the entries whose handle the tree holds at the end (n set_ttl calls in order)
    u64 set_batch_ttl(const char* blob, const u32* offsets, const u32* values, const u64* deadlines, u64 n);
    // removes up to `cap` topics whose handle's deadline is <= now, earliest first; their handles go to out[]
    u64 remove_expired(u64 now, u32* out, u64 cap);
    u32 dl_lookup_size() const { return dl_topic_.empty() ? 0u : static_cast<u32>(dl.size()); }   // 0: the lookup ignores deadlines
    std::vector<u64> dl;
    std::vector<u32> dirty_dl;
    bool full_dl = true;
    // n sets (start-up / restore: every retained message re-enters the tree, rmqtt-retainer/src/retainer.rs load path).
    // Returns the number of valid topics.  Into an EMPTY tree the host tree and its device image are built together, level
    // by level, on all host threads (set_batch_build); otherwise one by one.
    u64 set_batch(const char* blob, const u32* offsets, const u32* values, u64 n);

    // Dictionary compaction (HostTrie::compact): the level tokens this tree holds, and their replacement.
    std::vector<u32> used_tokens() const;
    void remap_tokens(const std::vector<u32>& remap);

    u64 values_size() const { return n_values_; }     // retain.rs:385-392
    u64 nodes_size() const { return n_nodes_; }       // retain.rs:395-398

    bool dirty = true;          // something to ship (whole arrays or patches)
    bool full = true;           // the arrays were rebuilt: ship them whole
    void prepare_flush();       // makes the arrays below current (flattens if in-place maintenance gave up)
    void shipped() { dirty = false; full = false; dirty_kids.clear(); dirty_edges.clear(); dirty_vals.clear(); dirty_dl.clear(); full_dl = false; }
    void flatten();                                     // host tree -> device-layout arrays below
    std::vector<RNode, HugeAlloc<RNode>> rnodes;        // host bookkeeping, one per device node (not shipped)
    std::vector<RKid, HugeAlloc<RKid>> rkids;
    ZeroTable<REdge> redges;                            // empty slot = all-zero bytes (child == 0)
    std::vector<u32, HugeAlloc<u32>> rvals;
    std::vector<u32> dirty_kids, dirty_edges, dirty_vals;   // entries changed in place since the last flush
    u32 root_plain_kids = 0, root_plain_val_hi = 0, max_depth = 0;
    u64 flattens = 0, patches = 0;                      // statistics: full rebuilds / in-place edits
    void debug_stats(uint64_t (&o)[6]) const { o[0] = flattens; o[1] = patches; o[2] = garbage_kids_; o[3] = dead_nodes_; o[4] = live_edges_; o[5] = flat_valid_ ? 1 : 0; }

  private:
    struct HN {
        std::vector<std::pair<u32, u32>> kids;   // (token, node), sorted by token
        u32 val = RVAL_NONE;
        bool has_val = false;
        u32 parent = 0, token = 0;
        u32 dev = RVAL_NONE;                     // device node of this host node (valid while flat_valid_)
    };
    // ---- in-place maintenance of the device image ----------------------------------------------
    static constexpr u32 NODEV = 0xFFFFFFFFu;
    bool flat_valid_ = false;                    // the arrays mirror the host tree (else: flatten at the next flush)
    BigVec<u32> rparent_, rtoken_, rcap_;        // per device node: parent, level token, capacity of its child block
    BigVec<u8> in_rvals_;                   // per device node: its value sits at rvals[val_lo] (it had one at flatten time)
    u64 garbage_kids_ = 0, dead_nodes_ = 0, live_edges_ = 0;
    void give_up() { flat_valid_ = false; dirty = true; }
    u32 edge_slot_of(u32 parent_dev, u32 token) const;          // slot in redges or NODEV
    void write_record(u32 dev);                                  // rnodes[dev] -> its two shipped copies
    void invalidate_ranges(u32 dev);                             // dev and its ancestors: walk instead of range-copy
    u32 dev_new_node(u32 parent_dev, u32 token);
    bool dev_add_child(u32 parent_dev, u32 token, u32 child_dev);
    void dev_set(u32 host_node, bool had_val, u32 value, u32 depth);
    void dev_unset(u32 host_node);
    u64 set_batch_build(const char* blob, const u32* offsets, const u32* values, u64 n, unsigned threads);
    int parse(const char* s, u32 len, bool create, std::vector<u32>& toks);
    u32 child_of(u32 node, u32 token) const;
    int put(const char* topic, u32 len, u32 value, bool* had_old, u32* old);
    bool holds(const char* topic, u32 len, u32 value);           // the topic's value is `value`
    void give_deadline(u32 h, const char* topic, u32 len, u64 deadline);
    void drop_deadline(u32 h);
    std::unordered_map<u32, std::string> dl_topic_;              // handle -> the topic it carries its deadline under
    std::vector<std::pair<u64, u32>> dl_heap_;                   // (deadline, handle), min-heap; stale once the handle's deadline changed
    HostTrie* dict_;
    BigVec<HN> nodes_;
    std::vector<u32> free_;
    std::vector<u32> toks_;
    u64 n_values_ = 0, n_nodes_ = 0;
};

}  // namespace gm
