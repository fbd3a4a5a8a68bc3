//! Raw bindings of `include/gpumqtt.h`.  UNTESTED SOURCE (no cargo in the image that built libgpumqtt.so).
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_void};

#[repr(C)]
pub struct gm_engine {
    _private: [u8; 0],
}

#[repr(C)]
#[derive(Clone, Copy)]
pub struct gm_config {
    pub struct_size: u32,
    pub device: i32,
    pub max_levels: u32,
    pub flags: u32,
    pub filters_hint: u64,
}

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct gm_span {
    pub off: u32,
    pub cnt: u32,
}

pub const GM_OK: i32 = 0;
pub const GM_ERR_INVALID_ARG: i32 = -1;
pub const GM_ERR_INVALID_TOPIC: i32 = -2;
pub const GM_ERR_CAPACITY: i32 = -3;
pub const GM_ERR_CUDA: i32 = -4;
pub const GM_ERR_TOO_DEEP: i32 = -5;
pub const GM_ERR_NO_DEVICE: i32 = -6;
pub const GM_ERR_TOO_LARGE: i32 = -7;
pub const GM_FLAG_MANUAL_FLUSH: u32 = 1;

#[link(name = "gpumqtt")]
extern "C" {
    pub fn gm_create(cfg: *const gm_config, out: *mut *mut gm_engine) -> i32;
    pub fn gm_destroy(e: *mut gm_engine);
    pub fn gm_last_error(e: *mut gm_engine) -> *const c_char;
    pub fn gm_version() -> *const c_char;
    pub fn gm_sub_add(e: *mut gm_engine, filter: *const u8, len: u32, value: u32, changed: *mut i32) -> i32;
    pub fn gm_sub_remove(e: *mut gm_engine, filter: *const u8, len: u32, value: u32, changed: *mut i32) -> i32;
    pub fn gm_bulk_load(e: *mut gm_engine, blob: *const u8, offsets: *const u32, values: *const u32, n: u64, n_changed: *mut u64) -> i32;
    pub fn gm_flush(e: *mut gm_engine) -> i32;
    pub fn gm_compact(e: *mut gm_engine) -> i32;
    pub fn gm_match_batch(
        e: *mut gm_engine, topics_blob: *const u8, topic_offsets: *const u32, n: u64, out_spans: *mut gm_span,
        out_ids: *mut u32, cap_ids: u64, needed: *mut u64, status: *mut i32,
    ) -> i32;
    pub fn gm_retain_set(e: *mut gm_engine, topic: *const u8, len: u32, value: u32, had_old: *mut i32, old_value: *mut u32) -> i32;
    pub fn gm_retain_remove(e: *mut gm_engine, topic: *const u8, len: u32, had_old: *mut i32, old_value: *mut u32) -> i32;
    pub fn gm_retain_bulk_load(e: *mut gm_engine, blob: *const u8, offsets: *const u32, values: *const u32, n: u64, n_set: *mut u64) -> i32;
    pub fn gm_retain_match_batch(
        e: *mut gm_engine, filters_blob: *const u8, filter_offsets: *const u32, n: u64, out_spans: *mut gm_span,
        out_ids: *mut u32, cap_ids: u64, needed: *mut u64, status: *mut i32,
    ) -> i32;
    pub fn gm_shard_of(topic_or_filter: *const u8, len: u32, n_shards: u32) -> u32;
    pub fn gm_shard_of_batch(blob: *const u8, offsets: *const u32, n: u64, n_shards: u32, out_shard: *mut u32) -> i32;
    pub fn gm_host_alloc(bytes: u64) -> *mut c_void;
    pub fn gm_host_free(p: *mut c_void);
}

// ---- round-2 additions of include/gpumqtt.h (same caveat: untested source) -------------------------------------------
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct gm_desc {
    pub r#ref: u32, // cnt == 1: the value itself; 2..65534: values[ref .. ref+cnt); 65535: ranges[ref]
    pub cnt: u32,
}
#[repr(C)]
pub struct gm_values {
    pub values: *const u32,
    pub n_values: u64,
    pub ranges: *const gm_span,
    pub n_ranges: u64,
    pub epoch: u64,
}
#[repr(C)]
pub struct gm_batcher {
    _private: [u8; 0],
}
pub type gm_match_cb = extern "C" fn(user: *mut c_void, cookie: u64, status: i32, ids: *const u32, n_ids: u32);
#[repr(C)]
pub struct gm_batcher_config {
    pub struct_size: u32,
    pub max_batch: u32,
    pub max_wait_us: u32,
    pub dispatchers: u32,
    pub on_match: gm_match_cb,
    pub user: *mut c_void,
}
extern "C" {
    pub fn gm_match_batch_desc(e: *mut gm_engine, topics_blob: *const u8, topic_offsets: *const u32, n: u64, out_spans: *mut gm_span,
                               out_descs: *mut gm_desc, cap_descs: u64, needed: *mut u64, status: *mut i32) -> i32;
    pub fn gm_values_view(e: *mut gm_engine, out: *mut gm_values) -> i32;
    pub fn gm_batcher_create(e: *mut gm_engine, cfg: *const gm_batcher_config, out: *mut *mut gm_batcher) -> i32;
    pub fn gm_submit(b: *mut gm_batcher, topic: *const u8, len: u32, cookie: u64) -> i32;
    pub fn gm_submit_publish(b: *mut gm_batcher, packet: *const u8, len: u32, cookie: u64) -> i32;
    pub fn gm_batcher_drain(b: *mut gm_batcher) -> i32;
    pub fn gm_batcher_destroy(b: *mut gm_batcher);
    /// A batcher over gm_retain_match_batch: gm_submit takes one SUBSCRIBE filter, the callback gets its retained handles.
    pub fn gm_retain_batcher_create(e: *mut gm_engine, cfg: *const gm_batcher_config, out: *mut *mut gm_batcher) -> i32;
    pub fn gm_sub_add_tree(e: *mut gm_engine, tree: u32, filter: *const u8, len: u32, value: u32, changed: *mut i32) -> i32;
    pub fn gm_sub_remove_tree(e: *mut gm_engine, tree: u32, filter: *const u8, len: u32, value: u32, changed: *mut i32) -> i32;
    pub fn gm_match_batch_trees(e: *mut gm_engine, topics_blob: *const u8, topic_offsets: *const u32, trees: *const u32, n: u64,
                                out_spans: *mut gm_span, out_ids: *mut u32, cap_ids: u64, needed: *mut u64, status: *mut i32) -> i32;
    pub fn gm_retain_remove_batch(e: *mut gm_engine, blob: *const u8, offsets: *const u32, n: u64, old_values: *mut u32, n_removed: *mut u64) -> i32;
    /// Expiry (RetainTree<TimedValue<Retain>>): deadlines in ms since the Unix epoch, 0 = none; expired iff now >= deadline.
    /// A handle with a deadline is stored under one topic only (a second one: GM_ERR_INVALID_ARG, nothing changed).
    pub fn gm_retain_set_ttl(e: *mut gm_engine, topic: *const u8, len: u32, value: u32, deadline_ms: u64, had_old: *mut i32, old_value: *mut u32) -> i32;
    pub fn gm_retain_bulk_load_ttl(e: *mut gm_engine, blob: *const u8, offsets: *const u32, values: *const u32, deadlines_ms: *const u64, n: u64,
                                   n_set: *mut u64) -> i32;
    /// gm_retain_match_batch at `now_ms` (gm_retain_match_batch itself uses the wall clock).
    pub fn gm_retain_match_batch_at(e: *mut gm_engine, now_ms: u64, filters_blob: *const u8, filter_offsets: *const u32, n: u64, out_spans: *mut gm_span,
                                    out_ids: *mut u32, cap_ids: u64, needed: *mut u64, status: *mut i32) -> i32;
    /// remove_expired_messages: up to `cap` expired topics in one lock acquisition; their handles go to out_values.
    pub fn gm_retain_remove_expired(e: *mut gm_engine, now_ms: u64, out_values: *mut u32, cap: u64, n_removed: *mut u64) -> i32;
}

// ---- the rest of include/gpumqtt.h: device-buffer entry points, router level, relation expansion, multi-GPU, probes ----
// (tests/test_abi.py::test_sys_crate_declares_every_function_of_the_header checks names and parameter counts against the header)
pub const GM_ERR_INTERNAL: i32 = -8;
pub const GM_ERR_COMM: i32 = -9;
pub const GM_FLAG_HOST_ONLY: u32 = 2;
pub const GM_FLAG_L2_FETCH_32: u32 = 4;
pub const GM_MATCH_DESCRIPTORS: u32 = 1;
pub const GM_COMM_ID_BYTES: usize = 128;
pub const GM_IPC_HANDLE_BYTES: usize = 64;
pub const GM_REL_LIVE: u32 = 1;
pub const GM_REL_V5: u32 = 2;
pub const GM_REL_NO_LOCAL: u32 = 4;
pub const GM_SUBREL_OFFLINE: u32 = 0x8000_0000;

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct gm_stats {
    pub values: u64,
    pub nodes: u64,
    pub device_nodes: u64,
    pub edges: u64,
    pub edge_slots: u64,
    pub dict_entries: u64,
    pub dict_slots: u64,
    pub plus_nodes: u64,
    pub value_words: u64,
    pub garbage_value_words: u64,
    pub device_bytes: u64,
    pub max_depth: u32,
    pub pending: u32,
    pub retained_values: u64,
    pub retained_nodes: u64,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct gm_work {
    pub visited: u64,
    pub probed: u64,
    pub filters: u64,
    pub ids: u64,
    pub levels: u64,
    pub bytes: u64,
    pub deferred: u64,
    pub probes_by_depth: [u64; 8],
    pub misses_by_depth: [u64; 8],
    pub slot_loads: u64,
}
#[repr(C)]
pub struct gm_match_args {
    pub struct_size: u32,
    pub flags: u32,
    pub d_blob: *const c_void,
    pub blob_bytes: u64,
    pub d_offsets: *const u32,
    pub n_entries: u64,
    pub d_sel: *const u32,
    pub n: u64,
    pub d_spans: *mut gm_span,
    pub d_out: *mut c_void,
    pub cap: u64,
    pub d_needed: *mut u64,
    pub d_status: *mut i32,
    pub stream: *mut c_void, // cudaStream_t
    pub work: *mut gm_work,
    pub d_trees: *const u32,
}
#[repr(C)]
pub struct gm_router {
    _private: [u8; 0],
}
#[repr(C)]
pub struct gm_id {
    pub node_id: u64,
    pub client_id: *const c_char,
    pub client_len: u32,
    pub _pad: u32,
    pub tag: u64,
}
#[repr(C)]
pub struct gm_sub_opts {
    pub qos: u8,
    pub is_v5: u8,
    pub no_local: u8,
    pub _pad: u8,
    pub sub_id: u32,
    pub shared_group: *const c_char,
    pub shared_group_len: u32,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct gm_sub_relation {
    pub node_id: u64,
    pub handle: u32,
    pub group: u32,
    pub sub_ids_off: u32,
    pub sub_ids_cnt: u32,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct gm_latency {
    pub p50_us: f64,
    pub p99_us: f64,
    pub mean_us: f64,
    pub max_us: f64,
    pub topics_per_s: f64,
    pub ids_per_topic: f64,
    pub samples: u64,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct gm_churn {
    pub seconds: f64,
    pub ops_per_s: f64,
    pub flushes_per_s: f64,
    pub mean_flush_us: f64,
    pub max_flush_us: f64,
    pub ops: u64,
    pub flushes: u64,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct gm_rel {
    pub node_id: u64,
    pub client_key: u32,
    pub id_idx: u32,
    pub sub_id: u32,
    pub flags: u32,
}
#[repr(C)]
pub struct gm_rel_out {
    pub d_spans: *mut gm_span,
    pub d_rels: *mut gm_sub_relation,
    pub cap_rels: u64,
    pub d_sub_ids: *mut u32,
    pub cap_sub_ids: u64,
    pub d_needed: *mut u64,
    pub d_status: *mut i32,
}
#[repr(C)]
pub struct gm_rel_groups {
    pub d_groups: *const gm_span,
    pub n_groups: u32,
    pub d_members: *const u32,
    pub d_online: *const u32,
    pub n_online_bits: u32,
    pub seed: u64,
}
#[repr(C)]
pub struct gm_gather_view {
    pub d_index: *const u32,
    pub d_spans: *const gm_span,
    pub d_ids: *const u32,
    pub d_counts: *const u64,
    pub slab_topics: u64,
    pub slab_ids: u64,
    pub world: u32,
    pub rank: u32,
}

extern "C" {
    // device-buffer forms of Router::matches / RetainStorage::get (asynchronous on a cudaStream_t)
    pub fn gm_match_batch_device(e: *mut gm_engine, d_topics_blob: *const c_void, blob_bytes: u64, d_topic_offsets: *const u32, n: u64,
                                 d_out_spans: *mut gm_span, d_out_ids: *mut u32, cap_ids: u64, d_needed: *mut u64, d_status: *mut i32,
                                 stream: *mut c_void) -> i32;
    pub fn gm_match_batch_device_stats(e: *mut gm_engine, d_topics_blob: *const c_void, blob_bytes: u64, d_topic_offsets: *const u32, n: u64,
                                       d_out_spans: *mut gm_span, d_out_ids: *mut u32, cap_ids: u64, d_needed: *mut u64, d_status: *mut i32,
                                       stream: *mut c_void, work: *mut gm_work) -> i32;
    pub fn gm_match_batch_device_ex(e: *mut gm_engine, a: *const gm_match_args) -> i32;
    pub fn gm_desc_expand(e: *mut gm_engine, descs: *const gm_desc, n: u64, out_ids: *mut u32, cap_ids: u64, needed: *mut u64) -> i32;
    pub fn gm_retain_match_batch_device(e: *mut gm_engine, d_filters_blob: *const c_void, blob_bytes: u64, d_filter_offsets: *const u32, n: u64,
                                        d_out_spans: *mut gm_span, d_out_ids: *mut u32, cap_ids: u64, needed: *mut u64, d_status: *mut i32,
                                        stream: *mut c_void) -> i32;
    // router level: DefaultRouter's relations, counters, Id rule, collector (rmqtt/src/router.rs:162-248, 417-479)
    pub fn gmr_create(e: *mut gm_engine, out: *mut *mut gm_router) -> i32;
    pub fn gmr_destroy(r: *mut gm_router);
    pub fn gmr_add(r: *mut gm_router, filter: *const u8, len: u32, id: *const gm_id, opts: *const gm_sub_opts) -> i32;
    pub fn gmr_remove(r: *mut gm_router, filter: *const u8, len: u32, id: *const gm_id, removed: *mut i32) -> i32;
    pub fn gmr_add_batch_numbered(r: *mut gm_router, blob: *const u8, offsets: *const u32, n: u64, node_ids: *const u64, client_nums: *const u32,
                                  flags: *const u8, sub_ids: *const u32, n_added: *mut u64) -> i32;
    pub fn gmr_last_timing(r: *mut gm_router, device_ms: *mut f64, host_ms: *mut f64) -> i32;
    pub fn gmr_topics(r: *mut gm_router) -> i64;
    pub fn gmr_routes(r: *mut gm_router) -> i64;
    pub fn gmr_matches_batch(r: *mut gm_router, publishers: *const gm_id, topics_blob: *const u8, topic_offsets: *const u32, n: u64,
                             out_spans: *mut gm_span, out_rels: *mut gm_sub_relation, cap_rels: u64, out_sub_ids: *mut u32, cap_sub_ids: u64,
                             needed_rels: *mut u64, needed_sub_ids: *mut u64, status: *mut i32) -> i32;
    pub fn gmr_matched_filters_batch(r: *mut gm_router, topics_blob: *const u8, topic_offsets: *const u32, n: u64, out_spans: *mut gm_span,
                                     out_filters: *mut u32, cap_filters: u64, needed: *mut u64, status: *mut i32) -> i32;
    pub fn gmr_filter(r: *mut gm_router, filter_idx: u32, filter: *mut *const c_char, filter_len: *mut u32, out_node_ids: *mut u64, cap_nodes: u32,
                      n_nodes: *mut u32) -> i32;
    pub fn gmr_relation(r: *mut gm_router, handle: u32, filter: *mut *const c_char, filter_len: *mut u32, client: *mut *const c_char,
                        client_len: *mut u32) -> i32;
    pub fn gmr_set_online(r: *mut gm_router, node_id: u64, client: *const c_char, len: u32, online: i32) -> i32;
    pub fn gmr_matches_batch_shared(r: *mut gm_router, seed: u64, publishers: *const gm_id, topics_blob: *const u8, topic_offsets: *const u32,
                                    n: u64, out_spans: *mut gm_span, out_rels: *mut gm_sub_relation, cap_rels: u64, out_sub_ids: *mut u32,
                                    cap_sub_ids: u64, needed_rels: *mut u64, needed_sub_ids: *mut u64, status: *mut i32) -> i32;
    pub fn gmr_group(r: *mut gm_router, group: u32, filter: *mut *const c_char, flen: *mut u32, name: *mut *const c_char, nlen: *mut u32,
                     out_handles: *mut u32, cap: u32, n: *mut u32) -> i32;
    // wire side + probes
    pub fn gm_publish_topic(packet: *const u8, len: u32, topic: *mut *const c_char, topic_len: *mut u32) -> i32;
    pub fn gm_batcher_probe(e: *mut gm_engine, blob: *const u8, offsets: *const u32, n: u64, burst: u32, rounds: u32, max_wait_us: u32,
                            out: *mut gm_latency) -> i32;
    pub fn gm_retain_batcher_probe(e: *mut gm_engine, blob: *const u8, offsets: *const u32, n: u64, burst: u32, rounds: u32, max_wait_us: u32,
                                   out: *mut gm_latency) -> i32;
    pub fn gm_churn_probe(e: *mut gm_engine, blob: *const u8, offsets: *const u32, values: *const u32, n: u64, target_ops_per_s: f64,
                          duration_ms: u32, flush_period_us: u32, out: *mut gm_churn) -> i32;
    // multi-GPU: communicator, device partition, the collective (NCCL form and the peer-memory form fused into the match kernels)
    pub fn gm_comm_unique_id(out_id: *mut u8) -> i32;
    pub fn gm_comm_init(e: *mut gm_engine, id: *const u8, rank: u32, world: u32) -> i32;
    pub fn gm_comm_destroy(e: *mut gm_engine) -> i32;
    pub fn gm_partition_batch_device(e: *mut gm_engine, d_blob: *const c_void, blob_bytes: u64, d_offsets: *const u32, n: u64, n_shards: u32,
                                     rank: u32, d_sel: *mut u32, d_shard: *mut u32, n_local: *mut u64, shard_counts: *mut u64,
                                     stream: *mut c_void) -> i32;
    pub fn gm_allgatherv_device(e: *mut gm_engine, d_index: *const u32, d_spans: *const gm_span, k: u64, d_ids: *const u32, d_m: *const u64,
                                d_all_index: *mut u32, d_all_spans: *mut gm_span, cap_topics: u64, d_all_ids: *mut u32, cap_ids: u64,
                                sizes: *mut u64, stream: *mut c_void) -> i32;
    pub fn gm_relations_expand_device(e: *mut gm_engine, d_spans: *const gm_span, d_ids: *const u32, n: u64, d_publishers: *const u32,
                                      d_rels: *const gm_rel, n_rels: u64, out: *const gm_rel_out, stream: *mut c_void) -> i32;
    pub fn gm_relations_choose_device(e: *mut gm_engine, d_spans: *const gm_span, d_ids: *const u32, n: u64, d_publishers: *const u32,
                                      d_rels: *const gm_rel, n_rels: u64, g: *const gm_rel_groups, out: *const gm_rel_out, stream: *mut c_void) -> i32;
    pub fn gm_share_key(seed: u64, row: u32, group: u32, occ: u32, client_key: u32) -> u64;
    pub fn gm_gather_create(e: *mut gm_engine, world: u32, rank: u32, slab_topics: u64, slab_ids: u64, out_handle: *mut u8) -> i32;
    pub fn gm_gather_connect(e: *mut gm_engine, handles: *const u8) -> i32;
    pub fn gm_match_gather_device(e: *mut gm_engine, d_blob: *const c_void, blob_bytes: u64, d_offsets: *const u32, n_entries: u64,
                                  d_sel: *const u32, n: u64, d_status: *mut i32, stream: *mut c_void) -> i32;
    pub fn gm_gather_get(e: *mut gm_engine, out: *mut gm_gather_view, stream: *mut c_void) -> i32;
    pub fn gm_gather_destroy(e: *mut gm_engine) -> i32;
    pub fn gm_device_read(e: *mut gm_engine, d_src: *const c_void, h_dst: *mut c_void, bytes: u64) -> i32;
    // introspection, diagnostics, NUMA placement
    pub fn gm_tokenize_batch(e: *mut gm_engine, topics_blob: *const u8, topic_offsets: *const u32, n: u64, max_tok: u32, out_tokens: *mut u32,
                             out_meta: *mut u32) -> i32;
    pub fn gm_get_stats(e: *mut gm_engine, out: *mut gm_stats) -> i32;
    pub fn gm_kernel_ms_ring(e: *mut gm_engine, out_ms: *mut f32, max_calls: u32, n_calls: *mut u32) -> i32;
    pub fn gm_kernel_launches(e: *mut gm_engine) -> u64;
    pub fn gm_debug_table(e: *mut gm_engine, which: u32, ptr: *mut *const c_void, count: *mut u64) -> i32;
    pub fn gm_debug_knob(e: *mut gm_engine, name: *const c_char, value: i64) -> i32;
    pub fn gm_host_alloc_near(e: *mut gm_engine, bytes: u64) -> *mut c_void;
    pub fn gm_device_numa_node(device: i32) -> i32;
    pub fn gm_bind_thread_near_device(device: i32) -> i32;
}

// ---- message store (rmqtt-message-storage's RAM backend with the forwarded marks on the device) ----
#[repr(C)]
pub struct gm_msgstore {
    _private: [u8; 0],
}

pub const GM_MSGSTORE_NO_SHARE: u32 = 0xFFFF_FFFF;

#[repr(C)]
#[derive(Clone, Copy)]
pub struct gm_msgstore_config {
    pub struct_size: u32,
    pub initial_mark_slots: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct gm_msgstore_stats {
    pub messages: u64,
    pub marks: u64,
    pub pending_marks: u64,
    pub mark_slots: u64,
    pub rehashes: u64,
    pub purges: u64,
    pub retired: u64,
}

extern "C" {
    /// gm_retain_match_batch_device at `now_ms`.
    pub fn gm_retain_match_batch_device_at(e: *mut gm_engine, now_ms: u64, d_filters_blob: *const c_void, blob_bytes: u64, d_filter_offsets: *const u32,
                                           n: u64, d_out_spans: *mut gm_span, d_out_ids: *mut u32, cap_ids: u64, needed: *mut u64, d_status: *mut i32,
                                           stream: *mut c_void) -> i32;
    /// The store owns its engine's retained tree: give it an engine of its own, with max_levels one above the broker's.
    pub fn gm_msgstore_create(e: *mut gm_engine, cfg: *const gm_msgstore_config, out: *mut *mut gm_msgstore) -> i32;
    pub fn gm_msgstore_destroy(ms: *mut gm_msgstore);
    /// _set: the message is kept under topic/<handle> until expiry_time_at_ms, marked as forwarded to (client_keys[i], share_keys[i]).
    pub fn gm_msgstore_store(ms: *mut gm_msgstore, topic: *const u8, len: u32, handle: u32, expiry_time_at_ms: u64, client_keys: *const u32,
                             share_keys: *const u32, n_marks: u32) -> i32;
    pub fn gm_msgstore_store_batch(ms: *mut gm_msgstore, blob: *const u8, offsets: *const u32, handles: *const u32, expiry_time_at_ms: *const u64, n: u64,
                                   mark_offsets: *const u32, client_keys: *const u32, share_keys: *const u32) -> i32;
    /// get for a batch of SUBSCRIBE filters, in batch order; returned messages are marked as forwarded to their query.
    pub fn gm_msgstore_get_batch(ms: *mut gm_msgstore, now_ms: u64, filters_blob: *const u8, filter_offsets: *const u32, n: u64, client_keys: *const u32,
                                 share_keys: *const u32, out_spans: *mut gm_span, out_handles: *mut u32, cap: u64, needed: *mut u64,
                                 status: *mut i32) -> i32;
    /// remove_expired_messages: expiry_time_at <= now_ms, earliest first; now_ms = u64::MAX - 1 evicts the `cap` earliest-expiring.
    pub fn gm_msgstore_remove_expired(ms: *mut gm_msgstore, now_ms: u64, out_handles: *mut u32, cap: u64, n_removed: *mut u64) -> i32;
    pub fn gm_msgstore_stats_get(ms: *mut gm_msgstore, out: *mut gm_msgstore_stats) -> i32;
}
