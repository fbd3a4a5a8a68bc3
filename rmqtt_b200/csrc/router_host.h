// GpuRouter — host-side mirror of rmqtt's DefaultRouter (rmqtt/src/router.rs:109-115) above the matching
// engine: the reference toolchain (Rust) is absent, so the Router-level semantics a Rust `GpuRouter` plugin
// would keep (INTEGRATION.md) are implemented here in C++ and driven through the gmr_* C entry points.
//
//   state     relations: filter -> client -> (Id, SubscriptionOptions)         router.rs:113  (AllRelationsMap, types.rs:443)
//             topics / routes counters                                          router.rs:112,114
//             the trie of the reference (`topics: TopicTree<()>`) is the device-resident trie of the engine;
//             its values are relation handles (one u32 per (filter, client))
//   add       router.rs:417-436        remove    router.rs:439-479 (Id-equality rule)
//   matches   router.rs:162-248 for a batch of PUBLISHes, ON THE DEVICE: engine match (gm_match_batch_device_ex) ->
//             k_relations (relations.cuh): no_local (:184-189), shared-group members passed through (:192-200),
//             v5 per-client de-dup with accumulation of subscription identifiers (types.rs:488-506) -> the host only
//             receives the finished gm_sub_relation records by DMA.  The router keeps a 24-byte gm_rel record per
//             handle in HBM (shipped incrementally).  matches_batch returns every shared-group member; with a seed
//             it chooses one per group on the device (k_relations<true>, subscribe.rs:66-104 with a seeded draw),
//             from per-group member blocks and an online bitmap the router keeps in device layout.  A topic with more
//             v5 relations than the kernel stages is de-duplicated by host_dedup_topic, by the kernel's rule: the
//             client's smallest handle represents it.
#pragma once
#include <algorithm>
#include <cstdint>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/gpumqtt.h"
#include "cuda_owned.h"

namespace gm {

class GpuRouter {
  public:
    struct Id { uint64_t node_id = 0; std::string client_id; uint64_t tag = 0;
                bool operator==(const Id& o) const { return node_id == o.node_id && tag == o.tag && client_id == o.client_id; } };   // types.rs:1746-1757
    struct Opts { uint8_t qos = 0, is_v5 = 0, no_local = 0; uint32_t sub_id = 0; std::string group; };                          // types.rs:565-718

    explicit GpuRouter(gm_engine* e) : e_(e) {}
    // timing of the last matches_batch call (milliseconds): device (H2D + match + relation kernel + D2H), host assembly
    double last_device_ms = 0, last_host_ms = 0;

    int32_t add(const char* filter, uint32_t len, const Id& id, const Opts& opts);
    int32_t remove(const char* filter, uint32_t len, const Id& id, bool* removed);
    int64_t topics() const { return topics_; }                // Router::topics  (router.rs:554-556)
    int64_t routes() const { return routes_; }                // Router::routes
    // share_seed: null returns every shared-group member; else one member per group is chosen with that seed
    int32_t matches_batch(const gm_id* publishers, const char* blob, const uint32_t* offs, uint64_t n, gm_span* out_spans,
                          gm_sub_relation* out_rels, uint64_t cap_rels, uint32_t* out_sub_ids, uint64_t cap_sub_ids,
                          uint64_t* needed_rels, uint64_t* needed_sub_ids, int32_t* status, const uint64_t* share_seed = nullptr);
    void set_online(uint64_t node_id, const std::string& client, bool online);        // Router::is_online
    bool group(uint32_t group, const std::string** filter, const std::string** name, const uint32_t** members, uint32_t* cnt) const;
    bool relation(uint32_t handle, const std::string** filter, const std::string** client) const;
    // unique matched filters per topic, through the engine's descriptor mode (router.rs:139-158, 315-363, 522-546)
    int32_t matched_filters_batch(const char* blob, const uint32_t* offs, uint64_t n, std::vector<gm_span>& spans, std::vector<uint32_t>& filters,
                                  std::vector<int32_t>& status);
    bool filter(uint32_t filter_idx, const std::string** name, std::vector<uint64_t>& node_ids) const;
    std::mutex mu;

  private:
    struct Rel { uint32_t filter_idx = 0; std::string client; Id id; Opts opts; bool live = false; };
    gm_engine* e_;
    std::unordered_map<std::string, uint32_t> filter_index_;
    std::vector<std::string> filter_names_;
    std::unordered_map<uint32_t, std::unordered_map<std::string, uint32_t>> relations_;   // filter idx -> client -> handle
    std::unordered_map<std::string, uint32_t> group_index_;                                // "filter\0group" -> 1-based id
    std::vector<Rel> by_handle_;
    std::vector<uint32_t> free_handles_;
    bool unflushed_removes_ = false;
    int64_t topics_ = 0, routes_ = 0;
    // ---- device side of the relation expansion ----
    std::vector<gm_rel> rel_host_;                                     // handle -> record, mirrored in HBM
    uint32_t rel_dirty_lo_ = 0xFFFFFFFFu, rel_dirty_hi_ = 0;           // handles changed since the last upload
    std::unordered_map<std::string, uint32_t> client_key_, id_idx_;    // "node\0client" -> key, "node\0client\0tag" -> idx
    DevBuf d_rels_;                                                    // shipped by dirty range: grows with its contents kept
    DevBuf d_blob_, d_offs_, d_spans_, d_status_, d_ids_, d_needed_, d_pubs_, d_ospans_, d_orels_, d_subs_;   // one call's scratch
    std::vector<uint32_t> pubs_;
    Stream stream_;                                                    // created by the first matches_batch
    // ---- shared groups in device layout (k_relations<true>): group id -> a block of live member handles with spare room in one
    //      pool; a block that fills up moves to the pool's end, and the pool is re-packed once the abandoned blocks pass half of it.
    //      The header, the pool and the online bitmap are shipped by dirty range, like rel_host_.
    struct Dirty { uint32_t lo = 0xFFFFFFFFu, hi = 0; void mark(uint32_t a, uint32_t b) { lo = std::min(lo, a); hi = std::max(hi, b); } bool any() const { return hi > lo; } };
    std::vector<gm_span> grp_hdr_{gm_span{0, 0}};                      // group id -> {off, cnt} in member_pool_; [0] unused
    std::vector<uint32_t> grp_cap_{0};                                 // group id -> block capacity
    std::vector<std::string> grp_filter_{std::string()}, grp_name_{std::string()};
    std::vector<uint32_t> member_pool_;
    std::vector<uint32_t> member_group_, member_slot_;                 // handle -> group it is listed in (0: none), its index in the block
    uint64_t pool_garbage_ = 0;
    Dirty hdr_dirty_, pool_dirty_, online_dirty_;                      // online_dirty_ counts words
    bool groups_changed_ = false;                                      // membership changed since the router's last gm_flush
    std::vector<uint32_t> online_words_;                               // bit per client_key, 1 = online
    DevBuf d_ghdr_, d_gmem_, d_online_;
    uint32_t intern(std::unordered_map<std::string, uint32_t>& m, const std::string& k) { return m.emplace(k, static_cast<uint32_t>(m.size())).first->second; }
    uint32_t client_key(uint64_t node_id, const std::string& client);
    void set_rel(uint32_t handle, const Rel& r);
    void member_add(uint32_t group, uint32_t handle);
    void member_remove(uint32_t handle);
    void repack_groups();
    int32_t ship_groups(cudaStream_t s);
    int32_t host_dedup_topic(const gm_sub_relation* in, uint32_t cnt, bool chosen, std::vector<gm_sub_relation>& rels, std::vector<uint32_t>& sub_ids);
};

}  // namespace gm
