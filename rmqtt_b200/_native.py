"""ctypes binding of libgpumqtt.so (include/gpumqtt.h).  Fails loudly when the library is missing:
there is no Python or CPU fallback for the matching path."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libgpumqtt.so"

GM_OK = 0
GM_ERR_INVALID_ARG = -1
GM_ERR_INVALID_TOPIC = -2
GM_ERR_CAPACITY = -3
GM_ERR_CUDA = -4
GM_ERR_TOO_DEEP = -5
GM_ERR_NO_DEVICE = -6
GM_ERR_TOO_LARGE = -7
GM_ERR_INTERNAL = -8
GM_ERR_COMM = -9
GM_MATCH_DESCRIPTORS = 1
GM_COMM_ID_BYTES = 128
GM_IPC_HANDLE_BYTES = 64
GM_FLAG_MANUAL_FLUSH = 1
GM_FLAG_HOST_ONLY = 2
GM_FLAG_L2_FETCH_32 = 4


class GmConfig(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("max_levels", C.c_uint32), ("flags", C.c_uint32),
                ("filters_hint", C.c_uint64)]


class GmStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("values", "nodes", "device_nodes", "edges", "edge_slots", "dict_entries",
                                           "dict_slots", "plus_nodes", "value_words", "garbage_value_words", "device_bytes")] + \
               [("max_depth", C.c_uint32), ("pending", C.c_uint32), ("retained_values", C.c_uint64), ("retained_nodes", C.c_uint64)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class GmId(C.Structure):
    _fields_ = [("node_id", C.c_uint64), ("client_id", C.c_char_p), ("client_len", C.c_uint32), ("_pad", C.c_uint32), ("tag", C.c_uint64)]


class GmSubOpts(C.Structure):
    _fields_ = [("qos", C.c_uint8), ("is_v5", C.c_uint8), ("no_local", C.c_uint8), ("_pad", C.c_uint8), ("sub_id", C.c_uint32),
                ("shared_group", C.c_char_p), ("shared_group_len", C.c_uint32)]


class GmSubRelation(C.Structure):
    _fields_ = [("node_id", C.c_uint64), ("handle", C.c_uint32), ("group", C.c_uint32), ("sub_ids_off", C.c_uint32), ("sub_ids_cnt", C.c_uint32)]


GM_SUBREL_OFFLINE = 0x80000000


class GmRelGroups(C.Structure):
    _fields_ = [("d_groups", C.c_void_p), ("n_groups", C.c_uint32), ("d_members", C.c_void_p), ("d_online", C.c_void_p),
                ("n_online_bits", C.c_uint32), ("seed", C.c_uint64)]


class GmWork(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("visited", "probed", "filters", "ids", "levels", "bytes", "deferred")] + \
               [("probes_by_depth", C.c_uint64 * 8), ("misses_by_depth", C.c_uint64 * 8), ("slot_loads", C.c_uint64)]

    def as_dict(self):
        d = {n: int(getattr(self, n)) for n in ("visited", "probed", "filters", "ids", "levels", "bytes", "deferred", "slot_loads")}
        d["probes_by_depth"] = [int(x) for x in self.probes_by_depth]
        d["misses_by_depth"] = [int(x) for x in self.misses_by_depth]
        return d


class GmMatchArgs(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("flags", C.c_uint32), ("d_blob", C.c_void_p), ("blob_bytes", C.c_uint64),
                ("d_offsets", C.c_void_p), ("n_entries", C.c_uint64), ("d_sel", C.c_void_p), ("n", C.c_uint64),
                ("d_spans", C.c_void_p), ("d_out", C.c_void_p), ("cap", C.c_uint64), ("d_needed", C.c_void_p), ("d_status", C.c_void_p),
                ("stream", C.c_void_p), ("work", C.POINTER(GmWork)), ("d_trees", C.c_void_p)]


class GmLatency(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("p50_us", "p99_us", "mean_us", "max_us", "topics_per_s", "ids_per_topic")] + [("samples", C.c_uint64)]

    def as_dict(self):
        return {n: float(getattr(self, n)) for n, _ in self._fields_[:-1]} | {"samples": int(self.samples)}


class GmChurn(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("seconds", "ops_per_s", "flushes_per_s", "mean_flush_us", "max_flush_us")] + [("ops", C.c_uint64), ("flushes", C.c_uint64)]

    def as_dict(self):
        return {n: (float(getattr(self, n)) if t is C.c_double else int(getattr(self, n))) for n, t in self._fields_}


GM_MATCH_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_uint64, C.c_int32, C.POINTER(C.c_uint32), C.c_uint32)


class GmBatcherConfig(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("max_batch", C.c_uint32), ("max_wait_us", C.c_uint32), ("dispatchers", C.c_uint32),
                ("on_match", GM_MATCH_CB), ("user", C.c_void_p)]


class GmGatherView(C.Structure):
    _fields_ = [("d_index", C.c_void_p), ("d_spans", C.c_void_p), ("d_ids", C.c_void_p), ("d_counts", C.c_void_p),
                ("slab_topics", C.c_uint64), ("slab_ids", C.c_uint64), ("world", C.c_uint32), ("rank", C.c_uint32)]


GM_MSGSTORE_NO_SHARE = 0xFFFFFFFF


class GmMsgstoreConfig(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("initial_mark_slots", C.c_uint32)]


class GmMsgstoreStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("messages", "marks", "pending_marks", "mark_slots", "rehashes", "purges", "retired")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class GmValues(C.Structure):
    _fields_ = [("values", C.c_void_p), ("n_values", C.c_uint64), ("ranges", C.c_void_p), ("n_ranges", C.c_uint64), ("epoch", C.c_uint64)]


# every symbol include/gpumqtt.h declares: name -> (restype, argtypes)
_vp, _cp, _u32, _u64, _i32 = C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint64, C.c_int32
_P = C.POINTER
SIGNATURES = {
    "gm_create": (_i32, [_P(GmConfig), _P(_vp)]),
    "gm_destroy": (None, [_vp]),
    "gm_last_error": (_cp, [_vp]),
    "gm_version": (_cp, []),
    "gm_sub_add": (_i32, [_vp, _cp, _u32, _u32, _P(_i32)]),
    "gm_sub_remove": (_i32, [_vp, _cp, _u32, _u32, _P(_i32)]),
    "gm_sub_add_tree": (_i32, [_vp, _u32, _cp, _u32, _u32, _P(_i32)]),
    "gm_sub_remove_tree": (_i32, [_vp, _u32, _cp, _u32, _u32, _P(_i32)]),
    "gm_match_batch_trees": (_i32, [_vp, _vp, _vp, _vp, _u64, _vp, _vp, _u64, _P(_u64), _vp]),
    "gm_bulk_load": (_i32, [_vp, _vp, _vp, _vp, _u64, _P(_u64)]),
    "gm_flush": (_i32, [_vp]),
    "gm_compact": (_i32, [_vp]),
    "gm_match_batch": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _u64, _P(_u64), _vp]),
    "gm_match_batch_device": (_i32, [_vp, _vp, _u64, _vp, _u64, _vp, _vp, _u64, _vp, _vp, _vp]),
    "gm_match_batch_device_stats": (_i32, [_vp, _vp, _u64, _vp, _u64, _vp, _vp, _u64, _vp, _vp, _vp, _P(GmWork)]),
    "gm_match_batch_device_ex": (_i32, [_vp, _P(GmMatchArgs)]),
    "gm_match_batch_desc": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _u64, _P(_u64), _vp]),
    "gm_values_view": (_i32, [_vp, _P(GmValues)]),
    "gm_desc_expand": (_i32, [_vp, _vp, _u64, _vp, _u64, _P(_u64)]),
    "gm_batcher_create": (_i32, [_vp, _P(GmBatcherConfig), _P(_vp)]),
    "gm_submit": (_i32, [_vp, _cp, _u32, _u64]),
    "gm_publish_topic": (_i32, [_vp, _u32, _P(_cp), _P(_u32)]),
    "gm_submit_publish": (_i32, [_vp, _vp, _u32, _u64]),
    "gm_batcher_drain": (_i32, [_vp]),
    "gm_batcher_destroy": (None, [_vp]),
    "gm_batcher_probe": (_i32, [_vp, _vp, _vp, _u64, _u32, _u32, _u32, _P(GmLatency)]),
    "gm_retain_batcher_create": (_i32, [_vp, _P(GmBatcherConfig), _P(_vp)]),
    "gm_retain_batcher_probe": (_i32, [_vp, _vp, _vp, _u64, _u32, _u32, _u32, _P(GmLatency)]),
    "gm_churn_probe": (_i32, [_vp, _vp, _vp, _vp, _u64, C.c_double, _u32, _u32, _P(GmChurn)]),
    "gm_relations_expand_device": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _u64, _vp, _vp]),
    "gm_relations_choose_device": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _u64, _P(GmRelGroups), _vp, _vp]),
    "gm_share_key": (_u64, [_u64, _u32, _u32, _u32, _u32]),
    "gm_gather_create": (_i32, [_vp, _u32, _u32, _u64, _u64, _vp]),
    "gm_gather_connect": (_i32, [_vp, _vp]),
    "gm_match_gather_device": (_i32, [_vp, _vp, _u64, _vp, _u64, _vp, _u64, _vp, _vp]),
    "gm_gather_get": (_i32, [_vp, _P(GmGatherView), _vp]),
    "gm_gather_destroy": (_i32, [_vp]),
    "gm_device_read": (_i32, [_vp, _vp, _vp, _u64]),
    "gm_comm_unique_id": (_i32, [_vp]),
    "gm_comm_init": (_i32, [_vp, _vp, _u32, _u32]),
    "gm_comm_destroy": (_i32, [_vp]),
    "gm_partition_batch_device": (_i32, [_vp, _vp, _u64, _vp, _u64, _u32, _u32, _vp, _vp, _P(_u64), _vp, _vp]),
    "gm_allgatherv_device": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp, _u64, _vp, _vp]),
    "gm_retain_set": (_i32, [_vp, _cp, _u32, _u32, _P(_i32), _P(_u32)]),
    "gm_retain_remove": (_i32, [_vp, _cp, _u32, _P(_i32), _P(_u32)]),
    "gm_retain_remove_batch": (_i32, [_vp, _vp, _vp, _u64, _vp, _P(_u64)]),
    "gm_retain_bulk_load": (_i32, [_vp, _vp, _vp, _vp, _u64, _P(_u64)]),
    "gm_retain_match_batch": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _u64, _P(_u64), _vp]),
    "gm_retain_match_batch_device": (_i32, [_vp, _vp, _u64, _vp, _u64, _vp, _vp, _u64, _P(_u64), _vp, _vp]),
    "gm_retain_set_ttl": (_i32, [_vp, _cp, _u32, _u32, _u64, _P(_i32), _P(_u32)]),
    "gm_retain_bulk_load_ttl": (_i32, [_vp, _vp, _vp, _vp, _vp, _u64, _P(_u64)]),
    "gm_retain_match_batch_at": (_i32, [_vp, _u64, _vp, _vp, _u64, _vp, _vp, _u64, _P(_u64), _vp]),
    "gm_retain_remove_expired": (_i32, [_vp, _u64, _vp, _u64, _P(_u64)]),
    "gm_retain_match_batch_device_at": (_i32, [_vp, _u64, _vp, _u64, _vp, _u64, _vp, _vp, _u64, _P(_u64), _vp, _vp]),
    "gm_msgstore_create": (_i32, [_vp, _P(GmMsgstoreConfig), _P(_vp)]),
    "gm_msgstore_destroy": (None, [_vp]),
    "gm_msgstore_store": (_i32, [_vp, _cp, _u32, _u32, _u64, _vp, _vp, _u32]),
    "gm_msgstore_store_batch": (_i32, [_vp, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp]),
    "gm_msgstore_get_batch": (_i32, [_vp, _u64, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _P(_u64), _vp]),
    "gm_msgstore_remove_expired": (_i32, [_vp, _u64, _vp, _u64, _P(_u64)]),
    "gm_msgstore_stats_get": (_i32, [_vp, _P(GmMsgstoreStats)]),
    "gmr_create": (_i32, [_vp, _P(_vp)]),
    "gmr_destroy": (None, [_vp]),
    "gmr_add": (_i32, [_vp, _cp, _u32, _P(GmId), _P(GmSubOpts)]),
    "gmr_remove": (_i32, [_vp, _cp, _u32, _P(GmId), _P(_i32)]),
    "gmr_add_batch_numbered": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _P(_u64)]),
    "gmr_last_timing": (_i32, [_vp, _P(C.c_double), _P(C.c_double)]),
    "gmr_topics": (C.c_int64, [_vp]),
    "gmr_routes": (C.c_int64, [_vp]),
    "gmr_matches_batch": (_i32, [_vp, _vp, _vp, _vp, _u64, _vp, _vp, _u64, _vp, _u64, _P(_u64), _P(_u64), _vp]),
    "gmr_matched_filters_batch": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _u64, _P(_u64), _vp]),
    "gmr_filter": (_i32, [_vp, _u32, _P(_cp), _P(_u32), _vp, _u32, _P(_u32)]),
    "gmr_relation": (_i32, [_vp, _u32, _P(_cp), _P(_u32), _P(_cp), _P(_u32)]),
    "gmr_set_online": (_i32, [_vp, _u64, _cp, _u32, _i32]),
    "gmr_matches_batch_shared": (_i32, [_vp, _u64, _vp, _vp, _vp, _u64, _vp, _vp, _u64, _vp, _u64, _P(_u64), _P(_u64), _vp]),
    "gmr_group": (_i32, [_vp, _u32, _P(_cp), _P(_u32), _P(_cp), _P(_u32), _vp, _u32, _P(_u32)]),
    "gm_tokenize_batch": (_i32, [_vp, _vp, _vp, _u64, _u32, _vp, _vp]),
    "gm_get_stats": (_i32, [_vp, _P(GmStats)]),
    "gm_kernel_ms_ring": (_i32, [_vp, _vp, _u32, _P(_u32)]),
    "gm_kernel_launches": (_u64, [_vp]),
    "gm_shard_of": (_u32, [_cp, _u32, _u32]),
    "gm_shard_of_batch": (_i32, [_vp, _vp, _u64, _u32, _vp]),
    "gm_debug_table": (_i32, [_vp, _u32, _P(_vp), _P(_u64)]),
    "gm_debug_knob": (_i32, [_vp, C.c_char_p, C.c_int64]),
    "gm_host_alloc": (_vp, [_u64]),
    "gm_host_alloc_near": (_vp, [_vp, _u64]),
    "gm_device_numa_node": (_i32, [_i32]),
    "gm_bind_thread_near_device": (_i32, [_i32]),
    "gm_host_free": (None, [_vp]),
}

_lib = None


def lib():
    """Loads libgpumqtt.so.  Raises if it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is None:
        import os
        path = Path(os.environ["GM_LIB"]) if os.environ.get("GM_LIB") else LIB_PATH      # A/B builds of the same library (tools/)
        if path != LIB_PATH and path.exists():
            L = C.CDLL(str(path))
            for name, (res, args) in SIGNATURES.items():
                f = getattr(L, name)
                f.restype, f.argtypes = res, args
            _lib = L
            return _lib
        if not LIB_PATH.exists():
            raise RuntimeError(f"{LIB_PATH} is missing: build it with __graft_entry__.build(); there is no fallback path")
        L = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib
