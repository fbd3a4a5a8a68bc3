/* libgpumqtt — C ABI of the H100-native (sm_90a) MQTT topic-filter matching engine.
 *
 * This is the drop-in boundary for ONE hot path of rmqtt (reference commit 4f9f2185):
 *
 *   Router::matches -> DefaultRouter::_matches -> TopicTree::matches      (PUBLISH, rmqtt/src/router.rs:162-248,
 *                                                                           rmqtt/src/trie.rs:143-145, 299-347)
 *   RetainStorage::get -> RetainTree::matches                              (SUBSCRIBE, rmqtt/src/retain.rs:152-169,
 *                                                                           291-367)
 *
 * A Rust plugin (`GpuRouter` / `GpuRetainer`, see INTEGRATION.md) keeps the reference's `Router` /
 * `RetainStorage` traits and forwards exactly these calls through `extern "C"`.  Plain pointers and
 * sizes only; no exceptions or aborts cross this boundary: every function returns a gm_status
 * (0 = ok, < 0 = error) and gm_last_error() gives the text.  Every handle is thread-safe (the
 * reference's objects are `Sync + Send`, router.rs:59).
 *
 * Values are u32 handles chosen by the caller (the host keeps handle -> (ClientId, Id, opts) /
 * handle -> Retain, i.e. today's `relations` DashMap and the retained payloads stay on the host).
 */
#ifndef GPUMQTT_H
#define GPUMQTT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gm_engine gm_engine;

typedef enum gm_status {
    GM_OK = 0,
    GM_ERR_INVALID_ARG = -1,
    GM_ERR_INVALID_TOPIC = -2, /* Topic::from_str would return Err (rmqtt/src/topic.rs:348-363) */
    GM_ERR_CAPACITY = -3,      /* out_ids too small; *needed tells how many ids the batch produces */
    GM_ERR_CUDA = -4,
    GM_ERR_TOO_DEEP = -5,      /* filter has more levels than gm_config.max_levels (cf. listener max_topic_levels, rmqtt/src/session.rs:1275) */
    GM_ERR_NO_DEVICE = -6,     /* no CUDA device: there is NO CPU fallback */
    GM_ERR_TOO_LARGE = -7,     /* batch exceeds a 32-bit offset (blob >= 4 GiB or ids >= 2^32) */
    GM_ERR_INTERNAL = -8,
    GM_ERR_COMM = -9           /* NCCL missing or a collective failed */
} gm_status;

typedef struct gm_config {
    uint32_t struct_size;      /* = sizeof(gm_config) */
    int32_t device;            /* CUDA device ordinal; -1 = current device */
    uint32_t max_levels;       /* deepest accepted filter (0 = default 128) */
    uint32_t flags;            /* GM_FLAG_* */
    uint64_t filters_hint;     /* expected number of filters (pre-sizes the tables), 0 = unknown */
} gm_config;

#define GM_FLAG_MANUAL_FLUSH 1u /* matches do NOT flush pending mutations implicitly (caller fences with gm_flush) */
#define GM_FLAG_L2_FETCH_32 4u  /* ask the CUDA context for 32-byte L2 fetches (cudaLimitMaxL2FetchGranularity): every hot access of the
                                   engine is a random 32-byte slot; the default 64-byte fetch wastes half the DRAM traffic.  Context-wide. */
#define GM_FLAG_HOST_ONLY 2u    /* staging mirror only, no CUDA context: add/remove/stats work, every match returns
                                   GM_ERR_NO_DEVICE (used by the CPU-side tests of the host logic) */

/* (offset, count) of one topic's result list inside out_ids */
typedef struct gm_span {
    uint32_t off;
    uint32_t cnt;
} gm_span;

typedef struct gm_stats {
    uint64_t values;           /* TopicTree::values_size  (rmqtt/src/trie.rs:148-151) — backs Router::topics_tree */
    uint64_t nodes;            /* TopicTree::nodes_size   (rmqtt/src/trie.rs:154-157) */
    uint64_t device_nodes;     /* node records resident on the device (includes pruned, not yet compacted ones) */
    uint64_t edges, edge_slots;
    uint64_t dict_entries, dict_slots;
    uint64_t plus_nodes;
    uint64_t value_words, garbage_value_words;
    uint64_t device_bytes;
    uint32_t max_depth;
    uint32_t pending;          /* 1 if mutations are staged and not yet flushed */
    uint64_t retained_values, retained_nodes;
} gm_stats;

/* exact work counters of the LAST gm_match_batch*_stats call — inputs of the roofline formula (DESIGN.md) */
typedef struct gm_work {
    uint64_t visited;          /* V: trie nodes visited  (MatchedIter::prepare calls) */
    uint64_t probed;           /* E: visited nodes with a non-empty remaining path */
    uint64_t filters;          /* F: matched filter nodes */
    uint64_t ids;              /* M: matched values */
    uint64_t levels;           /* L: topic levels */
    uint64_t bytes;            /* topic text bytes */
    uint64_t deferred;         /* topics handled by the generic (slow) kernel */
    uint64_t probes_by_depth[8]; /* diagnostics of the fast kernel: literal-child probes issued at depth d ... */
    uint64_t misses_by_depth[8]; /* ... of which the child did not exist */
    uint64_t slot_loads;         /* 32-byte edge-slot loads those probes cost (linear probing included) */
} gm_work;

/* ---- lifecycle -------------------------------------------------------------------------------------- */
int32_t gm_create(const gm_config* cfg, gm_engine** out);
void gm_destroy(gm_engine* e);
const char* gm_last_error(gm_engine* e); /* valid until the next call on `e` from the same thread */
const char* gm_version(void);

/* ---- subscription trie: TopicTree<u32>::insert / remove (rmqtt/src/trie.rs:99-135), driven by
 *      Router::add / Router::remove (rmqtt/src/router.rs:417-479).  `*changed` mirrors the reference's bool.
 *      Mutations are staged on the host and shipped to HBM by gm_flush (side stream).                     */
int32_t gm_sub_add(gm_engine* e, const char* filter, uint32_t len, uint32_t value, int32_t* changed);
int32_t gm_sub_remove(gm_engine* e, const char* filter, uint32_t len, uint32_t value, int32_t* changed);
/* Further TopicTree<V>s of the broker that are asked on every PUBLISH / SUBSCRIBE — ACL rule trees
 * (rmqtt-plugins/rmqtt-acl/src/config.rs:291-326, asked at rmqtt-acl/src/lib.rs:225,280), topic-rewrite rules
 * (rmqtt-topic-rewrite/src/lib.rs:138-155), bridge routing tables — live in the SAME engine as extra trie roots: `tree` 1..4095
 * names one (0 = the subscription trie; gm_sub_add == gm_sub_add_tree(0)).  A batch may mix rows of different trees
 * (gm_match_batch_trees / gm_match_args.d_trees): the PUBLISH match and its ACL check ride in one set of launches.
 * `is_match` (rmqtt/src/trie.rs:138-140) == the row's list is non-empty.  gm_get_stats counts all trees together.          */
int32_t gm_sub_add_tree(gm_engine* e, uint32_t tree, const char* filter, uint32_t len, uint32_t value, int32_t* changed);
int32_t gm_sub_remove_tree(gm_engine* e, uint32_t tree, const char* filter, uint32_t len, uint32_t value, int32_t* changed);
/* n filters at once (cluster restore re-inserts every filter, rmqtt-cluster-raft/src/router.rs:557-561).
 * Invalid filters are skipped; *n_changed = number of inserts that changed the tree.                      */
int32_t gm_bulk_load(gm_engine* e, const char* blob, const uint32_t* offsets /* n+1 */, const uint32_t* values,
                     uint64_t n, uint64_t* n_changed);
int32_t gm_flush(gm_engine* e);
/* Rebuilds the device tables from the live filters: drops the records of pruned nodes (rmqtt/src/trie.rs:126-128 removes
 * them eagerly; here they linger as dead records until compaction) and the garbage left by replaced value sets.
 * O(live filters + retained topics): the level dictionary is shared with the retained tree, whose nodes are re-labelled. */
int32_t gm_compact(gm_engine* e);

/* ---- Router::matches for a batch of PUBLISH topic names (host buffers).
 *      topics_blob/topic_offsets: n topic names back to back, topic i = blob[offsets[i] .. offsets[i+1]).
 *      out_spans[i] = where topic i's matched values sit in out_ids (multiset, order unspecified — the
 *      reference's order is hash-map iteration order too).  status[i] = GM_OK or GM_ERR_INVALID_TOPIC
 *      (that topic alone yields an empty list, like the per-call Err at rmqtt/src/router.rs:165).
 *      Returns GM_ERR_CAPACITY with *needed set when cap_ids is too small (nothing usable written).      */
int32_t gm_match_batch(gm_engine* e, const char* topics_blob, const uint32_t* topic_offsets, uint64_t n,
                       gm_span* out_spans, uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed,
                       int32_t* status);

/* gm_match_batch with a tree per row: topic i is matched against tree trees[i] (an unknown tree matches nothing). */
int32_t gm_match_batch_trees(gm_engine* e, const char* topics_blob, const uint32_t* topic_offsets, const uint32_t* trees, uint64_t n,
                             gm_span* out_spans, uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed, int32_t* status);

/* Same, with every buffer already in device memory, asynchronous on `stream` (a cudaStream_t).
 * d_needed (device u64) receives the number of ids produced; nothing is copied to the host.            */
int32_t gm_match_batch_device(gm_engine* e, const void* d_topics_blob, uint64_t blob_bytes,
                              const uint32_t* d_topic_offsets, uint64_t n, gm_span* d_out_spans,
                              uint32_t* d_out_ids, uint64_t cap_ids, uint64_t* d_needed, int32_t* d_status,
                              void* stream);
/* Instrumented variant of gm_match_batch_device: also accumulates the exact work counters (slower).    */
int32_t gm_match_batch_device_stats(gm_engine* e, const void* d_topics_blob, uint64_t blob_bytes,
                                    const uint32_t* d_topic_offsets, uint64_t n, gm_span* d_out_spans,
                                    uint32_t* d_out_ids, uint64_t cap_ids, uint64_t* d_needed,
                                    int32_t* d_status, void* stream, gm_work* work);

/* ---- general device-buffer entry point: descriptor output, selection of a sub-batch, work counters ----------------
 * d_blob must be readable in whole aligned 32-bit words (any cudaMalloc'd buffer or slice of one is).                */
#define GM_MATCH_DESCRIPTORS 1u   /* d_out receives gm_desc[] (one per matched FILTER) instead of u32 ids; cap / needed count descriptors */
typedef struct gm_desc {          /* reference to the value set of one matched filter node (rmqtt/src/trie.rs:70 BTreeSet<V>)             */
    uint32_t ref;                 /* cnt == 1: the value itself; 2 <= cnt < 65535: values[ref .. ref+cnt); cnt == 65535: ranges[ref] = {off, cnt} */
    uint32_t cnt;
} gm_desc;
typedef struct gm_match_args {
    uint32_t struct_size, flags;  /* = sizeof(gm_match_args); GM_MATCH_* */
    const void* d_blob; uint64_t blob_bytes;
    const uint32_t* d_offsets; uint64_t n_entries;   /* the packed batch: n_entries + 1 offsets */
    const uint32_t* d_sel;        /* NULL: match every entry (n = n_entries); else row t matches entry d_sel[t], t < n (a rank's share of a
                                     mixed batch, see gm_partition_batch_device) */
    uint64_t n;
    gm_span* d_spans; void* d_out; uint64_t cap; uint64_t* d_needed; int32_t* d_status;
    void* stream;
    gm_work* work;                /* optional: exact work counters (instrumented, slower; synchronises the stream) */
    const uint32_t* d_trees;      /* optional [n]: the tree every row is matched against (0 = the subscription trie), see gm_sub_add_tree */
} gm_match_args;
int32_t gm_match_batch_device_ex(gm_engine* e, const gm_match_args* a);

/* ---- descriptor mode with host buffers: what DefaultRouter::_matches consumes is one relations entry per matched filter
 *      (rmqtt/src/router.rs:166-182), so the engine can return the matched value SETS by reference (8 B per matched
 *      filter, ~4x less D2H traffic than 4 B per matched id) and the host reads the members from its own mirror.     */
int32_t gm_match_batch_desc(gm_engine* e, const char* topics_blob, const uint32_t* topic_offsets, uint64_t n,
                            gm_span* out_spans, gm_desc* out_descs, uint64_t cap_descs, uint64_t* needed, int32_t* status);
typedef struct gm_values {        /* host mirror of the value-set storage.  The two base pointers never change for the lifetime of
                                     the engine; entries a descriptor refers to stay intact while `epoch` is unchanged (mutations
                                     only append; gm_compact / automatic value compaction bump the epoch).                           */
    const uint32_t* values; uint64_t n_values;
    const gm_span* ranges; uint64_t n_ranges;        /* {off, cnt} of sets with >= 65535 members */
    uint64_t epoch;
} gm_values;
int32_t gm_values_view(gm_engine* e, gm_values* out);
/* convenience: expand descriptors into ids on the host (memcpy out of the mirror) */
int32_t gm_desc_expand(gm_engine* e, const gm_desc* descs, uint64_t n, uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed);

/* ---- retained-message tree: RetainTree<u32> (rmqtt/src/retain.rs:202-257), driven by RetainStorage::set
 *      (rmqtt-plugins/rmqtt-retainer/src/ram.rs:55-73 -> rmqtt/src/retain.rs:131-149: remove, then insert unless the
 *      payload is empty).  `value` is the caller's handle of the retained message; set replaces (Option::replace).  */
int32_t gm_retain_set(gm_engine* e, const char* topic, uint32_t len, uint32_t value, int32_t* had_old, uint32_t* old_value);
int32_t gm_retain_remove(gm_engine* e, const char* topic, uint32_t len, int32_t* had_old, uint32_t* old_value);
int32_t gm_retain_bulk_load(gm_engine* e, const char* blob, const uint32_t* offsets /* n+1 */, const uint32_t* values,
                            uint64_t n, uint64_t* n_set);
/* Batch removal under ONE lock acquisition — the expiry sweep (remove_expired_messages / RetainTree::retain,
 * rmqtt/src/retain.rs:118-128, 261-288: the host decides which retained topics expired).  old_values (optional, [n]) receives
 * the removed handle or 0xFFFFFFFF where nothing was stored; invalid topics are skipped.  A stored handle of 0xFFFFFFFF is
 * therefore indistinguishable from "nothing stored" in old_values: *n_removed is the count to trust.                          */
int32_t gm_retain_remove_batch(gm_engine* e, const char* blob, const uint32_t* offsets /* n+1 */, uint64_t n, uint32_t* old_values,
                               uint64_t* n_removed);
/* RetainStorage::get (rmqtt/src/retain.rs:152-169 -> RetainTree::matches :291-367) for a batch of SUBSCRIBE topic
 * FILTERS: out_spans[i] locates the handles of the retained messages filter i matches (order unspecified).
 * Same capacity / status protocol as gm_match_batch.                                                          */
int32_t gm_retain_match_batch(gm_engine* e, const char* filters_blob, const uint32_t* filter_offsets, uint64_t n,
                              gm_span* out_spans, uint32_t* out_ids, uint64_t cap_ids, uint64_t* needed, int32_t* status);
/* Same with device buffers on `stream`; synchronises the stream before returning (*needed is a host pointer). */
int32_t gm_retain_match_batch_device(gm_engine* e, const void* d_filters_blob, uint64_t blob_bytes,
                                     const uint32_t* d_filter_offsets, uint64_t n, gm_span* d_out_spans,
                                     uint32_t* d_out_ids, uint64_t cap_ids, uint64_t* needed, int32_t* d_status, void* stream);

/* ---- GpuRouter: DefaultRouter's Router-level semantics above the engine (rmqtt/src/router.rs:109-115, 162-248,
 *      417-479; rmqtt/src/types.rs:470-508).  This is what a Rust `GpuRouter` keeps on the host (INTEGRATION.md);
 *      it is provided in C++ because the reference toolchain is absent from the build image.                  */
typedef struct gm_router gm_router;
typedef struct gm_id {            /* rmqtt::types::Id; equality = all fields (types.rs:1746-1757): `tag` stands for lid/addrs/username/create_time */
    uint64_t node_id;
    const char* client_id;
    uint32_t client_len;
    uint32_t _pad;
    uint64_t tag;
} gm_id;
typedef struct gm_sub_opts {      /* rmqtt::types::SubscriptionOptions (types.rs:565-718) */
    uint8_t qos, is_v5, no_local, _pad;
    uint32_t sub_id;              /* v5 subscription identifier, 0 = none */
    const char* shared_group;     /* NULL / empty = not a shared subscription */
    uint32_t shared_group_len;
} gm_sub_opts;
typedef struct gm_sub_relation {  /* one element of SubRelations (types.rs:445-453) */
    uint64_t node_id;
    uint32_t handle;              /* -> (topic_filter, client_id) through gmr_relation */
    uint32_t group;               /* 0, or the id of the (filter, shared group) this member belongs to: the caller chooses one member */
    uint32_t sub_ids_off, sub_ids_cnt; /* v5: accumulated subscription identifiers in out_sub_ids */
} gm_sub_relation;
int32_t gmr_create(gm_engine* e, gm_router** out);   /* the router uses, but does not own, the engine */
void gmr_destroy(gm_router* r);
int32_t gmr_add(gm_router* r, const char* filter, uint32_t len, const gm_id* id, const gm_sub_opts* opts);   /* Router::add */
int32_t gmr_remove(gm_router* r, const char* filter, uint32_t len, const gm_id* id, int32_t* removed);       /* Router::remove */
/* Router::add for n subscriptions at once (snapshot restore, rmqtt-cluster-raft/src/router.rs:557-561) with numbered clients:
 * subscription i = (filter i, Id{node_ids[i], "c<client_nums[i]>", tag = client_nums[i]}, opts from flags[i] (bit 0 v5, bit 1 no_local)
 * and sub_ids[i]).  Invalid filters are skipped; *n_added counts the rest.                                                        */
int32_t gmr_add_batch_numbered(gm_router* r, const char* blob, const uint32_t* offsets, uint64_t n, const uint64_t* node_ids,
                               const uint32_t* client_nums, const uint8_t* flags, const uint32_t* sub_ids, uint64_t* n_added);
/* wall-clock split of the last gmr_matches_batch: device part (H2D, match + relation kernels, D2H) and host assembly, in ms */
int32_t gmr_last_timing(gm_router* r, double* device_ms, double* host_ms);
int64_t gmr_topics(gm_router* r);
int64_t gmr_routes(gm_router* r);
/* Router::matches for a batch; publishers[i] is the `this_id` of PUBLISH i (NULL: no no_local filtering).
 * Returns GM_ERR_CAPACITY with *needed_rels / *needed_sub_ids set when an output is too small.               */
int32_t gmr_matches_batch(gm_router* r, const gm_id* publishers, const char* topics_blob, const uint32_t* topic_offsets, uint64_t n,
                          gm_span* out_spans, gm_sub_relation* out_rels, uint64_t cap_rels, uint32_t* out_sub_ids, uint64_t cap_sub_ids,
                          uint64_t* needed_rels, uint64_t* needed_sub_ids, int32_t* status);
/* The secondary readers of the same tree — _has_matches (rmqtt/src/router.rs:139-142), _get_routes (:145-158), Router::get
 * (:522-546), _query_subscriptions_for_matches (:315-363) — all need the UNIQUE matched FILTERS of a topic.  Served by the
 * engine in descriptor mode (one descriptor per matched filter node; its first handle names the filter): out_spans[i] locates
 * topic i's unique matched filter indices in out_filters; gmr_filter gives a filter's string and the distinct node ids of its
 * relations.  No second CPU trie is needed for these calls.                                                                     */
int32_t gmr_matched_filters_batch(gm_router* r, const char* topics_blob, const uint32_t* topic_offsets, uint64_t n, gm_span* out_spans,
                                  uint32_t* out_filters, uint64_t cap_filters, uint64_t* needed, int32_t* status);
int32_t gmr_filter(gm_router* r, uint32_t filter_idx, const char** filter, uint32_t* filter_len, uint64_t* out_node_ids, uint32_t cap_nodes,
                   uint32_t* n_nodes);
int32_t gmr_relation(gm_router* r, uint32_t handle, const char** filter, uint32_t* filter_len, const char** client, uint32_t* client_len);

/* ---- single-call front end: Router::matches is called once per PUBLISH from many tokio workers (rmqtt/src/router.rs:482-484,
 *      caller rmqtt/src/shared.rs:601-636).  The batcher turns single submissions into device batches: a mutex-protected
 *      MPSC queue, a size / time window, `dispatchers` threads so that one batch is collected while others are on the device
 *      (the engine keeps several batches in flight and serves small ones as ONE CUDA-graph launch).  Completion is a
 *      callback per topic, from a dispatcher thread — a Rust caller completes a oneshot / writes an eventfd there.            */
typedef struct gm_batcher gm_batcher;
typedef void (*gm_match_cb)(void* user, uint64_t cookie, int32_t status, const uint32_t* ids, uint32_t n_ids);   /* ids valid during the call only */
typedef struct gm_batcher_config {
    uint32_t struct_size;      /* = sizeof(gm_batcher_config) */
    uint32_t max_batch;        /* dispatch when this many topics are queued (0 = default 4096) */
    uint32_t max_wait_us;      /* ... or when the oldest queued topic has waited this long */
    uint32_t dispatchers;      /* dispatch threads = batches in flight (0 = default 2) */
    gm_match_cb on_match;
    void* user;
} gm_batcher_config;
int32_t gm_batcher_create(gm_engine* e, const gm_batcher_config* cfg, gm_batcher** out);
int32_t gm_submit(gm_batcher* b, const char* topic, uint32_t len, uint64_t cookie);   /* thread-safe; never waits for the device */
/* Wire-side batching (SURVEY.md §8f-4): the topic name of a raw MQTT PUBLISH packet, zero-copy (*topic points into `packet`).
 * v3.1.1 and v5 share the layout — fixed header, remaining-length varint, u16-BE-prefixed topic (rmqtt-codec/src/v3/decode.rs:103-104,
 * rmqtt-codec/src/v5/packet/publish.rs:27-28).  gm_submit_publish feeds it to the batcher: the decoded topic bytes are the only
 * thing copied between the socket buffer and the device batch.  GM_ERR_INVALID_ARG: not a PUBLISH / malformed.                  */
int32_t gm_publish_topic(const uint8_t* packet, uint32_t len, const char** topic, uint32_t* topic_len);
int32_t gm_submit_publish(gm_batcher* b, const uint8_t* packet, uint32_t len, uint64_t cookie);
int32_t gm_batcher_drain(gm_batcher* b);                                              /* everything submitted so far has been delivered */
void gm_batcher_destroy(gm_batcher* b);
/* Closed-loop latency probe of that front end: `rounds` times, submit `burst` topics (taken cyclically from the packed batch)
 * one by one, wait until all their callbacks ran; per-topic latency = callback time - submit time.                             */
typedef struct gm_latency { double p50_us, p99_us, mean_us, max_us, topics_per_s, ids_per_topic; uint64_t samples; } gm_latency;
int32_t gm_batcher_probe(gm_engine* e, const char* blob, const uint32_t* offsets, uint64_t n, uint32_t burst, uint32_t rounds,
                         uint32_t max_wait_us, gm_latency* out);

/* Churn probe: remove + re-add the given (filter, value) pairs cyclically from the calling thread at `target_ops_per_s`
 * (0 = unthrottled) for `duration_ms`, with a gm_flush every `flush_period_us` (0 = leave it to the matches' auto-flush).
 * Run it in its own thread next to matching threads to measure mutation throughput and what it costs the matches.         */
typedef struct gm_churn { double seconds, ops_per_s, flushes_per_s, mean_flush_us, max_flush_us; uint64_t ops, flushes; } gm_churn;
int32_t gm_churn_probe(gm_engine* e, const char* blob, const uint32_t* offsets, const uint32_t* values, uint64_t n,
                       double target_ops_per_s, uint32_t duration_ms, uint32_t flush_period_us, gm_churn* out);

/* ---- multi-GPU (SURVEY.md §8e, BASELINE.json C5): one engine per GPU / process holds the filters of its root-hash shard
 *      (gm_shard_of; root-wildcard filters are replicated).  The host layer distributes the communicator id (in rmqtt: the
 *      cluster layer, rmqtt-plugins/rmqtt-cluster-raft; here torch.distributed or any channel).  libnccl is bound with
 *      dlopen at the first gm_comm_* call: GM_ERR_COMM when it is missing.                                                   */
#define GM_COMM_ID_BYTES 128
int32_t gm_comm_unique_id(uint8_t* out_id /* [GM_COMM_ID_BYTES] */);                 /* rank 0: ncclGetUniqueId */
int32_t gm_comm_init(gm_engine* e, const uint8_t* id, uint32_t rank, uint32_t world);  /* every rank, same id (collective) */
int32_t gm_comm_destroy(gm_engine* e);
/* Partition of a MIXED batch on the device: d_sel receives the entries whose root hashes to `rank` (order unspecified),
 * *n_local how many; optional d_shard[n] = shard of every entry, shard_counts[n_shards] (host) = load of every shard.
 * Feed d_sel / *n_local to gm_match_batch_device_ex.  Synchronises the stream (n_local is a host value).                   */
int32_t gm_partition_batch_device(gm_engine* e, const void* d_blob, uint64_t blob_bytes, const uint32_t* d_offsets, uint64_t n,
                                  uint32_t n_shards, uint32_t rank, uint32_t* d_sel, uint32_t* d_shard, uint64_t* n_local,
                                  uint64_t* shard_counts, void* stream);
/* The ONE collective of the path: all-gatherv of per-rank match lists, device buffers in, device buffers out, identical on
 * every rank.  Local contribution: k topics with global indices d_index[k] (= d_sel), d_spans[k] into d_ids[*d_m] (*d_m is the
 * DEVICE counter the match wrote: d_needed).  Output, rank-major: d_all_index / d_all_spans (re-based onto d_all_ids) /
 * d_all_ids; sizes[2*r] = topics, sizes[2*r+1] = ids of rank r (host array, 2*world).  ncclAllGather of the sizes + one
 * grouped launch of ncclSend/ncclRecv pairs reading the match kernels' own output buffers.  Collective: every rank must call it.
 * GM_ERR_CAPACITY when an output is too small (sizes[] is valid then).  Asynchronous on `stream` after one host sync.      */
int32_t gm_allgatherv_device(gm_engine* e, const uint32_t* d_index, const gm_span* d_spans, uint64_t k, const uint32_t* d_ids,
                             const uint64_t* d_m, uint32_t* d_all_index, gm_span* d_all_spans, uint64_t cap_topics,
                             uint32_t* d_all_ids, uint64_t cap_ids, uint64_t* sizes, void* stream);

/* ---- device-side relation expansion (SURVEY.md §8f-1): what DefaultRouter::_matches does with every matched relation after the
 *      trie walk — `no_local` (rmqtt/src/router.rs:184-189), pass-through of shared-group members (router.rs:192-200; the random
 *      pick of one member, :224-238, stays with the caller) and the per-client de-dup of v5 relations with accumulation of
 *      subscription identifiers (rmqtt/src/types.rs:488-506) — for a whole batch, on the match kernels' own device output.     */
typedef struct gm_rel {           /* one subscription relation, indexed by its handle (the value stored in the trie); 24 bytes */
    uint64_t node_id;             /* Id::node_id of the subscriber (SubRelationsMap is keyed by it, rmqtt/src/types.rs:466) */
    uint32_t client_key;          /* index of the (node id, client id) pair: the v5 de-dup key */
    uint32_t id_idx;              /* index of the subscriber's full Id: no_local compares Ids (types.rs:1746-1757) */
    uint32_t sub_id;              /* v5 subscription identifier, 0 = none */
    uint32_t flags;               /* GM_REL_* | shared-group id << 8 (0 = not a shared subscription) */
} gm_rel;
#define GM_REL_LIVE 1u
#define GM_REL_V5 2u
#define GM_REL_NO_LOCAL 4u
typedef struct gm_rel_out {
    gm_span* d_spans;             /* [n] per topic: its relations in d_rels */
    gm_sub_relation* d_rels; uint64_t cap_rels;      /* finished records: node id, handle, group, sub-id range */
    uint32_t* d_sub_ids; uint64_t cap_sub_ids;
    uint64_t* d_needed;           /* device [3]: relations, sub ids produced, (unused) — capacity protocol: compare on the host, retry */
    int32_t* d_status;            /* [n]: set to 1 where a topic had more v5 relations than the kernel stages (256): that topic's list is
                                     complete but NOT de-duplicated — the caller finishes it */
} gm_rel_out;
/* d_spans / d_ids: the output of gm_match_batch_device* (ids mode); d_publishers[n]: id_idx of every PUBLISH's sender or 0xFFFFFFFF
 * (NULL: no no_local filtering); d_rels[n_rels]: the relation table.  Asynchronous on `stream`.                                   */
int32_t gm_relations_expand_device(gm_engine* e, const gm_span* d_spans, const uint32_t* d_ids, uint64_t n, const uint32_t* d_publishers,
                                   const gm_rel* d_rels, uint64_t n_rels, const gm_rel_out* out, void* stream);

/* ---- the same exchange FUSED into the match kernels over peer memory (NVLink / NVSwitch): the publish phase of the match writes
 *      every topic's span, global index and ids directly into the gathered arrays of ALL ranks while the walk of the next tiles is
 *      still running — no separate collective, no host synchronisation; a one-warp kernel ends the step with the contribution
 *      counts and a flag barrier.  Layout: every rank owns one device block with a fixed SLAB per rank (slab_topics rows, slab_ids
 *      ids): rank r's rows are [r * slab_topics, r * slab_topics + counts[2r]) of d_index / d_spans (spans are absolute offsets
 *      into d_ids, rank r's ids start at r * slab_ids).  Needs peer-to-peer access between the GPUs (CUDA IPC): gm_gather_connect
 *      returns GM_ERR_COMM where that is unavailable — use gm_allgatherv_device (NCCL) there.  world <= 8.                         */
#define GM_IPC_HANDLE_BYTES 64
int32_t gm_gather_create(gm_engine* e, uint32_t world, uint32_t rank, uint64_t slab_topics, uint64_t slab_ids,
                         uint8_t* out_handle /* [GM_IPC_HANDLE_BYTES]: give it to every other rank */);
int32_t gm_gather_connect(gm_engine* e, const uint8_t* handles /* [world][GM_IPC_HANDLE_BYTES], rank order */);
/* match this rank's rows (d_sel / n as in gm_match_args) and publish into every rank's block.  Collective in effect: every rank
 * calls it once per step; asynchronous on `stream`; when the stream has passed it on a rank, ALL ranks' results are in its block. */
int32_t gm_match_gather_device(gm_engine* e, const void* d_blob, uint64_t blob_bytes, const uint32_t* d_offsets, uint64_t n_entries,
                               const uint32_t* d_sel, uint64_t n, int32_t* d_status, void* stream);
typedef struct gm_gather_view {
    const uint32_t* d_index; const gm_span* d_spans; const uint32_t* d_ids;
    const uint64_t* d_counts;     /* device [world][2]: rows, ids contributed by every rank in the last step */
    uint64_t slab_topics, slab_ids; uint32_t world, rank;
} gm_gather_view;
int32_t gm_gather_get(gm_engine* e, gm_gather_view* out, void* stream);   /* synchronises `stream`; GM_ERR_COMM if a rank missed the barrier */
int32_t gm_gather_destroy(gm_engine* e);
int32_t gm_device_read(gm_engine* e, const void* d_src, void* h_dst, uint64_t bytes);   /* convenience: device -> host copy (tests, tools) */

/* ---- tokeniser only (Topic::from_str for a batch) — used by tests to pin the device dictionary.
 *      out_tokens: [max_tok][n] u32 (level-major), out_meta: [n] (bits 0..23 levels, bit 30 '$', bit 31 invalid) */
int32_t gm_tokenize_batch(gm_engine* e, const char* topics_blob, const uint32_t* topic_offsets, uint64_t n,
                          uint32_t max_tok, uint32_t* out_tokens, uint32_t* out_meta);

/* ---- misc ------------------------------------------------------------------------------------------- */
int32_t gm_get_stats(gm_engine* e, gm_stats* out);
/* device time (ms) of the three kernels — [0] tokenise [1] match [2] deferred — of the last <= 64 match calls
 * (either entry point), oldest first, measured with CUDA events on the stream the kernels ran on.
 * out_ms holds 3*max_calls floats; *n_calls receives how many calls were written.  Synchronises on them. */
int32_t gm_kernel_ms_ring(gm_engine* e, float* out_ms, uint32_t max_calls, uint32_t* n_calls);
/* number of kernels the engine has launched since creation */
uint64_t gm_kernel_launches(gm_engine* e);
/* shard of a topic / filter by its level-0 string (multi-GPU root-hash partitioning); 0xFFFFFFFF for a
 * filter whose level 0 is a wildcard (those are replicated on every shard)                               */
uint32_t gm_shard_of(const char* topic_or_filter, uint32_t len, uint32_t n_shards);
/* the same for a packed batch (blob + n+1 offsets): out_shard[i] = gm_shard_of(entry i); pure host function          */
int32_t gm_shard_of_batch(const char* blob, const uint32_t* offsets, uint64_t n, uint32_t n_shards, uint32_t* out_shard);
/* DEBUG/TEST: read-only view of the host mirror of a device table, in device layout (rmqtt_b200/csrc/layout.h).
 * which: 0 edges(32 B) 2 ranges(8 B) 3 values(4 B) 4 dict(32 B) 5 long-string pool(1 B)
 *        6 root record {plus, hash_ref, mask, max_depth, hash_cnt, win_mask, win_shift, nwin_mask}; retained tree: 7 nodes(32 B, host bookkeeping) 8 child blocks(32 B entries)
 *        9 pre-order values(4 B); 10 (parent, token) hash slots (32 B); 11 maintenance counters (6 x u64: full rebuilds, in-place
 *        patches, garbage child entries, dead nodes, hash entries, image valid); 12 child filter of wide nodes (4 B words).  Valid until the next mutating call.                                       */
int32_t gm_debug_table(gm_engine* e, uint32_t which, const void** ptr, uint64_t* count);
/* DEBUG/TUNING: set a kernel-scheduling knob of this engine at run time (A/B measurements; results never change).
 * "tile_chunk" (1..1024: consecutive 32-topic tiles a CTA of the match kernel reserves at once), "k2_ctas" (0 = default),
 * "sorted_rows" (0/1), "bucket_bits" (100*a+b: locality buckets = 2^(a+b)), "diag_flags" (timing diagnostics: see kernels.cuh MP_DIAG_*; results are WRONG when set).       */
int32_t gm_debug_knob(gm_engine* e, const char* name, int64_t value);
/* pinned host memory for the host-buffer entry points */
void* gm_host_alloc(uint64_t bytes);
/* the same, placed on the NUMA node the engine's GPU hangs off (its PCIe root): on a 2-socket server a pinned buffer on
 * the far socket crosses the inter-socket link on every copy.  Falls back to gm_host_alloc placement without NUMA info. */
void* gm_host_alloc_near(gm_engine* e, uint64_t bytes);
int32_t gm_device_numa_node(int32_t device);            /* -1 unknown */
/* restricts the CALLING thread (and threads it creates later) to the CPUs of the GPU's NUMA node and prefers that
 * node for its allocations — what each per-GPU worker of a multi-GPU host should do once at start                      */
int32_t gm_bind_thread_near_device(int32_t device);
void gm_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif /* GPUMQTT_H */
