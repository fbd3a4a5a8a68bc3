// Data layout shared by the host mirror (host_trie.cpp) and the sm_90a kernels (kernels.cuh).
//
// The reference keeps the subscription trie as HashMap<Level, Node> per node with a BTreeSet<V> of
// values (rmqtt/src/trie.rs:69-73).  Here the whole trie lives in HBM as four flat arrays:
//
//   dict   : open-addressing table  level string -> u32 token          (32-B slots, string inline)
//   edges  : open-addressing table  (parent node, token) -> child + the child's *node record*
//            (32-B slots; ONE 32-byte load answers "does the child exist, what are its values, its
//             '#'-child values, its '+'-child, which tokens can continue below it")
//   ranges / values : value sets with >1 element (single values are stored inline in the record)
//
// A node record = {plus, hash_ref, own_ref, mask}:
//   plus     1 + the slot of `edges` that holds this node's '+' child (0 = none): the '+' hop is a direct
//            load of that slot, no hashing                                      trie.rs:330-334
//   hash_ref value set of this node's '#' child (with its 16-bit count in cnts)   trie.rs:302-308,321-327
//   own_ref  value set of the node itself                                        trie.rs:309-310
//   mask     bits 0..22: Bloom mask over the tokens of all children (skips hopeless literal probes)
//            bit 23: wide node (its child edges are registered in the child filter, below)
//            bits 24..31: window tag — which WINDOW of the edge table holds this node's child edges (below)
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define GM_HD __host__ __device__ __forceinline__
#else
#define GM_HD inline
#endif

namespace gm {

using u8 = uint8_t;
using u32 = uint32_t;
using u64 = uint64_t;

// ---- tokens -----------------------------------------------------------------------------------
constexpr u32 TOK_UNKNOWN = 0;  // level string not in the dictionary: no literal child can match
constexpr u32 TOK_PLUS = 1;     // "+"  (Level::SingleWildcard)
constexpr u32 TOK_HASH = 2;     // "#"  (Level::MultiWildcard)
constexpr u32 TOK_BLANK = 3;    // ""   (Level::Blank)
constexpr u32 TOK_FIRST = 4;    // first dictionary-assigned token

// ---- value-set references -----------------------------------------------------------------------
// A value set (BTreeSet<V> of one trie node, trie.rs:70) is published as (ref, cnt16):
//   cnt == 0            empty
//   cnt == 1            ref IS the value                       (no second memory access)
//   2 <= cnt < CNT_BIG  values[ref .. ref+cnt)                 (contiguous, coalesced copy)
//   cnt == CNT_BIG      ranges[ref] = {off, cnt}: a set of >= 65535 values (deferred path only)
constexpr u32 CNT_BIG = 0xFFFFu;

struct alignas(32) EdgeSlot {
    u32 parent;    // key
    u32 token;     // key
    u32 child;     // node id of the child; 0 = empty slot (node ids start at 1, the root is 0)
    u32 plus;      // record of `child` ...
    u32 hash_ref;
    u32 own_ref;
    u32 mask;
    u32 cnts;      // hash_cnt | own_cnt << 16
};
static_assert(sizeof(EdgeSlot) == 32, "EdgeSlot must be one 32-byte sector");

// Dictionary slot: w[0] = token (0 = empty).  Inline strings (<= 27 bytes): bytes 4..30 = the string, zero
// padded, byte 31 = its length — i.e. w[1..7] are exactly the words the tokeniser packs, so a lookup is
// seven word compares.  Long strings: byte 31 = 0xFF, w[1] = length, w[2] = offset into the long-string
// pool, w[3] = FNV-1a hash of all bytes.
struct alignas(32) DictSlot {
    u32 w[8];
};
static_assert(sizeof(DictSlot) == 32, "DictSlot must be one 32-byte sector");
constexpr u32 DICT_INLINE_MAX = 27;

struct Range { u32 off, cnt; };

// ---- child filter of wide nodes -----------------------------------------------------------------
// The 32-bit Bloom mask in a record saturates once a node has more than a few dozen children, yet exactly
// those nodes (`reg/+`, `+/site`, ...) are probed by every topic for children that mostly do not exist —
// each such probe is a cold HBM request that finds an empty slot (measured: 1.76 M of them per 1 M topics on
// C3).  Nodes with more than WIDE_FANOUT literal children therefore register ALL their child edges in one
// small blocked Bloom filter (16 bits per edge; a few MB, L2 resident) and announce it with a flag in the
// mask word of their record.  A negative answer skips the probe; stale bits after removals
// only cost a wasted probe.
constexpr u32 MASK_WIDE_FLAG = 1u << 23;
constexpr u32 WIDE_FANOUT = 48;


// ---- windows of the edge table -------------------------------------------------------------------
// Random 32-B fetches from a multi-GB table run faster when each CTA stays inside a window of <= 64 MiB
// (address-translation reach) than when every SM roams the whole table.  The edge table is therefore cut into `nwin` equal
// windows (a power of two): the child edges of a node all live in ONE window, named by the 8-bit tag in the
// node's record; trie nodes of depth >= 3 inherit the tag of their depth-2 ancestor, so a whole
// `level0/level1/...` subtree hashes into one window — and since the batch is walked in (level0, level1)
// order (k_bucket_*), the cold probes of neighbouring topics land in the same few windows.  The children of
// the root and of its children live in window 0 (hot, L2 resident).  Effective window = tag & (nwin-1), so
// the host can halve `nwin` (one subtree outgrew its window) or grow the table without re-tagging.
constexpr u32 MASK_BLOOM_BITS = 23;
constexpr u32 MASK_BLOOM = (1u << MASK_BLOOM_BITS) - 1u;
constexpr u32 WTAG_SHIFT = 24;
constexpr u32 WTAG_COUNT = 256;          // tags are assigned over the full 8-bit range
constexpr u32 WIN_MIN_SLOTS_LOG2 = 12;   // never cut windows smaller than 4096 slots (128 KiB)
constexpr u32 WIN_MAX_LOG2 = 8;          // at most 256 windows

// Root record + table geometry handed to every kernel by value.
struct TrieView {
    const EdgeSlot* edges;
    const Range* ranges;
    const u32* values;
    const DictSlot* dict;
    const u8* pool;
    const u32* cfilter;     // child filter of wide nodes (words)
    u32 cfilter_mask;       // #words - 1
    u32 edge_mask;      // capacity-1 (capacity is a power of two)
    u32 win_mask;       // slots per window - 1
    u32 win_shift;      // log2(slots per window)
    u32 nwin_mask;      // windows - 1
    u32 dict_mask;
    u32 root_plus, root_hash_ref, root_hash_cnt, root_mask;
    u32 max_depth;      // deepest filter in the trie (levels)
    const u32* tree_slots;  // extra trees of the engine (ACL rules, rewrite rules, ...): tree id -> edge slot of its root record
    u32 n_trees;            // entries in tree_slots (index 0 unused: tree 0's root record travels above)
};

// Per-topic word written by the tokeniser: bits 0..23 level count, bit 30 level 0 is Metadata ('$...'),
// bit 31 Topic::from_str would fail (topic.rs:348-363) -> the topic matches nothing.
constexpr u32 META_INVALID = 0x80000000u;
constexpr u32 META_DOLLAR = 0x40000000u;
constexpr u32 META_NLEV_MASK = 0x00FFFFFFu;

// ---- hashing (identical on host and device) -----------------------------------------------------
GM_HD u32 fmix32(u32 h) {
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
    return h;
}
GM_HD u32 edge_hash(u32 parent, u32 token) {
    return fmix32(parent * 0x9E3779B1u + (token ^ 0x7F4A7C15u) * 0x85EBCA77u);
}
constexpr u32 FNV_INIT = 0x811C9DC5u;
GM_HD u32 fnv_step(u32 h, u32 byte) { return (h ^ byte) * 0x01000193u; }
GM_HD u32 dict_hash_finish(u32 h, u32 len) { return fmix32(h ^ (len * 0x9E3779B1u)); }   // long strings: h = FNV-1a over bytes
// inline strings: hash of the seven packed key words (length included in the last one)
GM_HD u32 dict_hash_words(const u32 (&w)[7]) {
    u32 h = FNV_INIT;
    for (int k = 0; k < 7; ++k) h = (h ^ w[k]) * 0x01000193u;
    return fmix32(h);
}
GM_HD u32 mask_bit(u32 token) { return 1u << ((((token * 0x9E3779B1u) >> 16) * MASK_BLOOM_BITS) >> 16); }   // one of 23 bits
// first slot of the probe sequence of edge (parent, token) whose parent carries window tag `wtag`, and the
// successor of a slot: linear probing that wraps inside the window
GM_HD u32 edge_slot0(u32 parent, u32 token, u32 wtag, u32 win_mask, u32 win_shift, u32 nwin_mask) {
    return ((wtag & nwin_mask) << win_shift) | (edge_hash(parent, token) & win_mask);
}
GM_HD u32 edge_next(u32 idx, u32 win_mask) { return (idx & ~win_mask) | ((idx + 1u) & win_mask); }
// child filter of wide nodes: word index + the two bits of an edge
GM_HD void cfilter_pos(u32 parent, u32 token, u32 word_mask, u32& word, u32& bits) {
    const u32 h = fmix32((parent ^ 0x68E31DA4u) * 0x9E3779B1u + token * 0x85EBCA77u);
    const u32 g = fmix32(h + 0x9E3779B9u);
    word = h & word_mask;
    bits = (1u << (g & 31u)) | (1u << ((g >> 5) & 31u));
}

// Shard of a level-0 string (multi-GPU partitioning by topic root, SURVEY §8e).
GM_HD u32 shard_of_hash(u32 h, u32 nshards) { return static_cast<u32>((static_cast<u64>(fmix32(h ^ 0x5bd1e995u)) * nshards) >> 32); }

}  // namespace gm
