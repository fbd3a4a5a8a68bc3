"""Host-side handle over the C ABI (include/gpumqtt.h).

`Engine` is the Python face of one `gm_engine`: the device-resident subscription trie with the
`TopicTree<u32>` operations of the reference (`insert` / `remove` / `matches`,
rmqtt/src/trie.rs:99-145) applied to whole batches.  Everything that matches runs in the CUDA
library; if libgpumqtt.so or a CUDA device is missing the calls raise — there is no fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N


class GpuMqttError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libgpumqtt error {code}: {msg}")
        self.code = code


def _b(s) -> bytes:
    return s if isinstance(s, (bytes, bytearray)) else s.encode("utf-8")


def _vp(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def pack(strings):
    """list[str|bytes] -> (blob uint8[], offsets uint32[n+1])"""
    bs = [_b(s) for s in strings]
    offs = np.zeros(len(bs) + 1, dtype=np.uint32)
    if bs:
        offs[1:] = np.cumsum([len(b) for b in bs], dtype=np.uint64).astype(np.uint32)
    blob = np.frombuffer(b"".join(bs), dtype=np.uint8).copy() if bs else np.zeros(0, np.uint8)
    return blob, offs


class MatchResult:
    """Per-topic match lists: topic i -> ids[spans[i,0] : spans[i,0]+spans[i,1]] (multiset, unordered)."""

    def __init__(self, spans: np.ndarray, ids: np.ndarray, status: np.ndarray, needed: int):
        self.spans, self.ids, self.status, self.needed = spans, ids, status, needed

    def __len__(self):
        return len(self.spans)

    def sorted_list(self, i: int):
        """Sorted multiset of topic i, or None if the topic is invalid (reference: Err)."""
        if self.status[i] != 0:
            return None
        off, cnt = int(self.spans[i, 0]), int(self.spans[i, 1])
        return sorted(self.ids[off:off + cnt].tolist())

    def counts(self) -> np.ndarray:
        c = self.spans[:, 1].astype(np.int64)
        c[self.status != 0] = -1
        return c

    def canonical(self):
        """(counts int64[n] with -1 for invalid, ids sorted within each topic, concatenated in topic order)."""
        counts = self.counts()
        n = len(counts)
        pos = np.maximum(counts, 0)
        starts = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(pos, out=starts[1:])
        total = int(starts[-1])
        if total == 0:
            return counts, np.zeros(0, dtype=np.uint32)
        # gather each topic's ids into topic order, then sort within segments via a (segment, id) lexsort
        seg = np.repeat(np.arange(n, dtype=np.int64), pos)
        within = np.arange(total, dtype=np.int64) - np.repeat(starts[:-1], pos)
        src = np.repeat(self.spans[:, 0].astype(np.int64), pos) + within
        vals = self.ids[src]
        order = np.lexsort((vals, seg))
        return counts, vals[order]


class Engine:
    def __init__(self, device: int = -1, max_levels: int = 0, manual_flush: bool = False, filters_hint: int = 0,
                 host_only: bool = False):
        self._lib = N.lib()
        flags = (N.GM_FLAG_MANUAL_FLUSH if manual_flush else 0) | (N.GM_FLAG_HOST_ONLY if host_only else 0)
        cfg = N.GmConfig(C.sizeof(N.GmConfig), device, max_levels, flags, filters_hint)
        h = C.c_void_p()
        rc = self._lib.gm_create(C.byref(cfg), C.byref(h))
        if rc != N.GM_OK:
            raise GpuMqttError(rc, self._lib.gm_last_error(None).decode())
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.gm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != N.GM_OK:
            raise GpuMqttError(rc, self._lib.gm_last_error(self._h).decode())

    # ---- TopicTree::insert / remove ---------------------------------------------------------------
    def add(self, filt, value: int) -> bool:
        b = _b(filt)
        ch = C.c_int32(0)
        self._check(self._lib.gm_sub_add(self._h, b, len(b), value, C.byref(ch)))
        return bool(ch.value)

    def remove(self, filt, value: int) -> bool:
        b = _b(filt)
        ch = C.c_int32(0)
        self._check(self._lib.gm_sub_remove(self._h, b, len(b), value, C.byref(ch)))
        return bool(ch.value)

    # ---- further TopicTree<V>s in the same engine (ACL rule trees, rewrite rules, ...): extra trie roots ------------
    def add_tree(self, tree: int, filt, value: int) -> bool:
        b = _b(filt)
        ch = C.c_int32(0)
        self._check(self._lib.gm_sub_add_tree(self._h, tree, b, len(b), value, C.byref(ch)))
        return bool(ch.value)

    def remove_tree(self, tree: int, filt, value: int) -> bool:
        b = _b(filt)
        ch = C.c_int32(0)
        self._check(self._lib.gm_sub_remove_tree(self._h, tree, b, len(b), value, C.byref(ch)))
        return bool(ch.value)

    def match_batch_trees(self, blob: np.ndarray, offs: np.ndarray, trees: np.ndarray) -> MatchResult:
        """Row i is matched against tree trees[i] (0 = the subscription trie): mixed batches in one set of launches."""
        n = len(offs) - 1
        trees = np.ascontiguousarray(trees, dtype=np.uint32)
        assert len(trees) == n
        spans = np.zeros((n, 2), dtype=np.uint32)
        status = np.zeros(n, dtype=np.int32)
        cap = max(1024, 32 * n)
        while True:
            ids = np.empty(cap, dtype=np.uint32)
            needed = C.c_uint64(0)
            rc = self._lib.gm_match_batch_trees(self._h, _vp(blob), _vp(offs), _vp(trees), n, _vp(spans), _vp(ids), cap, C.byref(needed), _vp(status))
            if rc == N.GM_ERR_CAPACITY:
                cap = int(needed.value)
                continue
            self._check(rc)
            return MatchResult(spans, ids[:int(needed.value)], status, int(needed.value))

    def bulk_load(self, blob: np.ndarray, offs: np.ndarray, values: np.ndarray) -> int:
        assert blob.dtype == np.uint8 and offs.dtype == np.uint32 and values.dtype == np.uint32
        n_changed = C.c_uint64(0)
        self._check(self._lib.gm_bulk_load(self._h, _vp(blob), _vp(offs), _vp(values), len(values), C.byref(n_changed)))
        return int(n_changed.value)

    def flush(self):
        self._check(self._lib.gm_flush(self._h))

    def compact(self):
        self._check(self._lib.gm_compact(self._h))

    # ---- Router::matches for a batch (host buffers) ---------------------------------------------------
    def match_batch(self, blob: np.ndarray, offs: np.ndarray, cap_ids: int | None = None) -> MatchResult:
        assert blob.dtype == np.uint8 and offs.dtype == np.uint32
        n = len(offs) - 1
        spans = np.zeros((n, 2), dtype=np.uint32)
        status = np.zeros(n, dtype=np.int32)
        cap = int(cap_ids) if cap_ids is not None else max(1024, 32 * n)
        while True:
            ids = np.empty(cap, dtype=np.uint32)
            needed = C.c_uint64(0)
            rc = self._lib.gm_match_batch(self._h, _vp(blob), _vp(offs), n, _vp(spans), _vp(ids), cap, C.byref(needed), _vp(status))
            if rc == N.GM_ERR_CAPACITY and cap_ids is None:
                cap = int(needed.value)
                continue
            self._check(rc)
            return MatchResult(spans, ids[:int(needed.value)], status, int(needed.value))

    def match_topics(self, topics, cap_ids: int | None = None) -> MatchResult:
        blob, offs = pack(topics)
        return self.match_batch(blob, offs, cap_ids)

    def matches(self, topic):
        """TopicTree::matches for one topic -> sorted multiset (None if invalid)."""
        return self.match_topics([topic]).sorted_list(0)

    # ---- retained-message tree: RetainTree insert / remove / matches (rmqtt/src/retain.rs) ------------------
    def retain_set(self, topic, value: int):
        """Returns the replaced value or None."""
        b = _b(topic)
        had, old = C.c_int32(0), C.c_uint32(0)
        self._check(self._lib.gm_retain_set(self._h, b, len(b), value, C.byref(had), C.byref(old)))
        return int(old.value) if had.value else None

    def retain_remove(self, topic):
        b = _b(topic)
        had, old = C.c_int32(0), C.c_uint32(0)
        self._check(self._lib.gm_retain_remove(self._h, b, len(b), C.byref(had), C.byref(old)))
        return int(old.value) if had.value else None

    def retain_remove_batch(self, blob: np.ndarray, offs: np.ndarray):
        """-> (old handles uint32[n] with 0xFFFFFFFF where nothing was stored, number removed).  A stored handle of
        0xFFFFFFFF looks the same as "nothing stored" in the first array; the number removed is the count to trust."""
        n = len(offs) - 1
        old = np.empty(n, dtype=np.uint32)
        cnt = C.c_uint64(0)
        self._check(self._lib.gm_retain_remove_batch(self._h, _vp(blob), _vp(offs), n, _vp(old), C.byref(cnt)))
        return old, int(cnt.value)

    def retain_bulk_load(self, blob: np.ndarray, offs: np.ndarray, values: np.ndarray) -> int:
        n_set = C.c_uint64(0)
        self._check(self._lib.gm_retain_bulk_load(self._h, _vp(blob), _vp(offs), _vp(values), len(values), C.byref(n_set)))
        return int(n_set.value)

    def retain_match_batch(self, blob: np.ndarray, offs: np.ndarray, cap_ids: int | None = None) -> MatchResult:
        n = len(offs) - 1
        spans = np.zeros((n, 2), dtype=np.uint32)
        status = np.zeros(n, dtype=np.int32)
        cap = int(cap_ids) if cap_ids is not None else max(1024, 64 * n)
        while True:
            ids = np.empty(cap, dtype=np.uint32)
            needed = C.c_uint64(0)
            rc = self._lib.gm_retain_match_batch(self._h, _vp(blob), _vp(offs), n, _vp(spans), _vp(ids), cap, C.byref(needed), _vp(status))
            if rc == N.GM_ERR_CAPACITY and cap_ids is None:
                cap = int(needed.value)
                continue
            self._check(rc)
            return MatchResult(spans, ids[:int(needed.value)], status, int(needed.value))

    def retain_matches(self, filt):
        blob, offs = pack([filt])
        return self.retain_match_batch(blob, offs).sorted_list(0)

    def retain_match_batch_device(self, d_blob, d_offs, d_spans, d_ids, d_status, stream: int) -> int:
        n = d_offs.numel() - 1
        needed = C.c_uint64(0)
        self._check(self._lib.gm_retain_match_batch_device(self._h, d_blob.data_ptr(), d_blob.numel(), d_offs.data_ptr(), n, d_spans.data_ptr(),
                                                           d_ids.data_ptr(), d_ids.numel(), C.byref(needed), d_status.data_ptr(), stream))
        return int(needed.value)

    # ---- device-resident variant (torch tensors; asynchronous on the current torch stream) -----------
    def match_batch_device(self, d_blob, d_offs, d_spans, d_ids, d_needed, d_status, stream: int, work: bool = False):
        n = d_offs.numel() - 1
        args = [self._h, d_blob.data_ptr(), d_blob.numel(), d_offs.data_ptr(), n, d_spans.data_ptr(), d_ids.data_ptr(),
                d_ids.numel(), d_needed.data_ptr(), d_status.data_ptr(), stream]
        if work:
            w = N.GmWork()
            self._check(self._lib.gm_match_batch_device_stats(*args, C.byref(w)))
            return w.as_dict()
        self._check(self._lib.gm_match_batch_device(*args))
        return None

    def match_batch_device_ex(self, d_blob, d_offs, d_spans, d_out, d_needed, d_status, stream: int, *, desc: bool = False, d_sel=None,
                              n_sel: int | None = None, work: bool = False):
        """gm_match_batch_device_ex: descriptor output (d_out = int64/uint2 tensor of gm_desc) and / or a selection of rows."""
        n_entries = d_offs.numel() - 1
        n = n_entries if d_sel is None else int(n_sel)
        w = N.GmWork() if work else None
        elem = 8 if desc else 4
        a = N.GmMatchArgs(C.sizeof(N.GmMatchArgs), N.GM_MATCH_DESCRIPTORS if desc else 0, d_blob.data_ptr(), d_blob.numel(), d_offs.data_ptr(), n_entries,
                          d_sel.data_ptr() if d_sel is not None else None, n, d_spans.data_ptr(), d_out.data_ptr(),
                          d_out.numel() * d_out.element_size() // elem, d_needed.data_ptr(), d_status.data_ptr(), stream,
                          C.pointer(w) if work else None)
        self._check(self._lib.gm_match_batch_device_ex(self._h, C.byref(a)))
        return w.as_dict() if work else None

    # ---- descriptor mode (host buffers): matched value SETS by reference --------------------------------------
    def match_batch_desc(self, blob: np.ndarray, offs: np.ndarray, cap: int | None = None):
        """-> (spans uint32[n,2] into descs, descs uint32[m,2] = (ref, cnt), status, needed)"""
        n = len(offs) - 1
        spans = np.zeros((n, 2), dtype=np.uint32)
        status = np.zeros(n, dtype=np.int32)
        c = int(cap) if cap is not None else max(1024, 16 * n)
        while True:
            descs = np.empty((c, 2), dtype=np.uint32)
            needed = C.c_uint64(0)
            rc = self._lib.gm_match_batch_desc(self._h, _vp(blob), _vp(offs), n, _vp(spans), _vp(descs), c, C.byref(needed), _vp(status))
            if rc == N.GM_ERR_CAPACITY and cap is None:
                c = int(needed.value)
                continue
            self._check(rc)
            return spans, descs[:int(needed.value)], status, int(needed.value)

    def values_view(self):
        """Zero-copy numpy views of the host mirror of the value-set storage: (values uint32[], ranges uint32[k,2], epoch)."""
        v = N.GmValues()
        self._check(self._lib.gm_values_view(self._h, C.byref(v)))
        vals = np.frombuffer((C.c_uint32 * int(v.n_values)).from_address(v.values), dtype=np.uint32) if v.n_values else np.zeros(0, np.uint32)
        rng = np.frombuffer((C.c_uint32 * (2 * int(v.n_ranges))).from_address(v.ranges), dtype=np.uint32).reshape(-1, 2) if v.n_ranges else np.zeros((0, 2), np.uint32)
        return vals, rng, int(v.epoch)

    def desc_expand(self, descs: np.ndarray) -> np.ndarray:
        descs = np.ascontiguousarray(descs, dtype=np.uint32)
        n = len(descs)
        needed = C.c_uint64(0)
        cap = int(descs[:, 1].astype(np.int64).sum()) + 1024 if n else 1
        while True:
            out = np.empty(cap, dtype=np.uint32)
            rc = self._lib.gm_desc_expand(self._h, _vp(descs), n, _vp(out), cap, C.byref(needed))
            if rc == N.GM_ERR_CAPACITY:
                cap = int(needed.value)
                continue
            self._check(rc)
            return out[:int(needed.value)]

    def match_batch_via_desc(self, blob: np.ndarray, offs: np.ndarray) -> "MatchResult":
        """Descriptor-mode match expanded on the host (gm_desc_expand) into the MatchResult shape of match_batch (tests)."""
        spans, descs, status, _ = self.match_batch_desc(blob, offs)
        _, rng, _ = self.values_view()
        cnt = descs[:, 1].astype(np.int64)
        big = cnt == 0xFFFF
        if big.any():
            cnt[big] = rng[descs[big, 0], 1]
        starts = np.zeros(len(descs) + 1, dtype=np.int64)
        np.cumsum(cnt, out=starts[1:])
        ids = self.desc_expand(descs)                 # ids in descriptor order; a topic's descriptors are contiguous
        assert len(ids) == int(starts[-1])
        d0 = spans[:, 0].astype(np.int64)
        d1 = d0 + spans[:, 1].astype(np.int64)
        ispans = np.stack([starts[d0], starts[d1] - starts[d0]], axis=1)
        return MatchResult(ispans.astype(np.uint32), ids, status, len(ids))

    # ---- multi-GPU: communicator, device partition, all-gatherv (include/gpumqtt.h, comm.cuh) --------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * N.GM_COMM_ID_BYTES)()
        rc = N.lib().gm_comm_unique_id(buf)
        if rc != N.GM_OK:
            raise GpuMqttError(rc, N.lib().gm_last_error(None).decode())
        return bytes(buf)

    def comm_init(self, uid: bytes, rank: int, world: int):
        buf = (C.c_uint8 * N.GM_COMM_ID_BYTES).from_buffer_copy(uid)
        self._check(self._lib.gm_comm_init(self._h, buf, rank, world))
        self._world = world

    def partition_batch_device(self, d_blob, d_offs, n_shards: int, rank: int, d_sel, stream: int, d_shard=None):
        """-> (n_local, shard_counts int64[n_shards])"""
        n = d_offs.numel() - 1
        n_local = C.c_uint64(0)
        counts = np.zeros(n_shards, dtype=np.uint64)
        self._check(self._lib.gm_partition_batch_device(self._h, d_blob.data_ptr(), d_blob.numel(), d_offs.data_ptr(), n, n_shards, rank, d_sel.data_ptr(),
                                                        d_shard.data_ptr() if d_shard is not None else None, C.byref(n_local), _vp(counts), stream))
        return int(n_local.value), counts.astype(np.int64)

    def allgatherv_device(self, d_index, d_spans, k: int, d_ids, d_m, d_all_index, d_all_spans, d_all_ids, stream: int):
        """-> sizes int64[world, 2] = (topics, ids) contributed by every rank"""
        sizes = np.zeros(2 * self._world, dtype=np.uint64)
        self._check(self._lib.gm_allgatherv_device(self._h, d_index.data_ptr() if d_index is not None else None, d_spans.data_ptr(), k, d_ids.data_ptr(), d_m.data_ptr(),
                                                   d_all_index.data_ptr(), d_all_spans.data_ptr(), d_all_index.numel(), d_all_ids.data_ptr(), d_all_ids.numel(),
                                                   _vp(sizes), stream))
        return sizes.astype(np.int64).reshape(-1, 2)

    # ---- fused gather over peer memory (the match kernels publish straight into every rank's gathered arrays) -----------
    def gather_create(self, world: int, rank: int, slab_topics: int, slab_ids: int) -> bytes:
        buf = (C.c_uint8 * N.GM_IPC_HANDLE_BYTES)()
        self._check(self._lib.gm_gather_create(self._h, world, rank, slab_topics, slab_ids, buf))
        self._gworld = world
        return bytes(buf)

    def gather_connect(self, handles):
        """handles: list of `world` byte strings in rank order (this rank's own entry is ignored)."""
        blob = b"".join(handles)
        assert len(blob) == self._gworld * N.GM_IPC_HANDLE_BYTES
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        self._check(self._lib.gm_gather_connect(self._h, buf))

    def match_gather_device(self, d_blob, d_offs, d_status, stream: int, d_sel=None, n_sel: int | None = None):
        n_entries = d_offs.numel() - 1
        n = n_entries if d_sel is None else int(n_sel)
        self._check(self._lib.gm_match_gather_device(self._h, d_blob.data_ptr(), d_blob.numel(), d_offs.data_ptr(), n_entries,
                                                     d_sel.data_ptr() if d_sel is not None else None, n, d_status.data_ptr(), stream))

    def gather_result(self, stream: int):
        """Synchronises and copies this rank's gathered block to the host:
        -> (counts int64[world,2], index uint32[K], spans uint32[K,2] (absolute into ids), ids uint32[world*slab_ids])"""
        v = N.GmGatherView()
        self._check(self._lib.gm_gather_get(self._h, C.byref(v), stream))
        W, T, I = int(v.world), int(v.slab_topics), int(v.slab_ids)
        counts = np.zeros((W, 2), dtype=np.uint64)
        self._check(self._lib.gm_device_read(self._h, v.d_counts, _vp(counts), counts.nbytes))
        idx = np.zeros(W * T, dtype=np.uint32); sp = np.zeros((W * T, 2), dtype=np.uint32); ids = np.zeros(W * I, dtype=np.uint32)
        self._check(self._lib.gm_device_read(self._h, v.d_index, _vp(idx), idx.nbytes))
        self._check(self._lib.gm_device_read(self._h, v.d_spans, _vp(sp), sp.nbytes))
        self._check(self._lib.gm_device_read(self._h, v.d_ids, _vp(ids), ids.nbytes))
        rows = np.concatenate([np.arange(r * T, r * T + int(counts[r, 0])) for r in range(W)]) if W else np.zeros(0, np.int64)
        return counts.astype(np.int64), idx[rows], sp[rows], ids

    def gather_destroy(self):
        self._check(self._lib.gm_gather_destroy(self._h))

    # ---- tokeniser hook -------------------------------------------------------------------------------
    def tokenize(self, topics, max_tok: int = 16):
        blob, offs = pack(topics)
        n = len(offs) - 1
        toks = np.zeros((max_tok, n), dtype=np.uint32)
        meta = np.zeros(n, dtype=np.uint32)
        self._check(self._lib.gm_tokenize_batch(self._h, _vp(blob), _vp(offs), n, max_tok, _vp(toks), _vp(meta)))
        return toks, meta

    # ---- introspection -----------------------------------------------------------------------------------
    def stats(self) -> dict:
        s = N.GmStats()
        self._check(self._lib.gm_get_stats(self._h, C.byref(s)))
        return s.as_dict()

    def debug_tables(self) -> dict:
        """Host mirror of the device tables as numpy arrays (copies).  Test/diagnostic use only."""
        out = {}
        spec = {0: ("edges", np.uint32, 8), 2: ("ranges", np.uint32, 2), 3: ("values", np.uint32, 1),
                4: ("dict", np.uint32, 8), 5: ("pool", np.uint8, 1), 6: ("root", np.uint32, 1),  # root = {plus, hash_ref, mask, max_depth, hash_cnt, win_mask, win_shift, nwin_mask}
                7: ("rnodes", np.uint32, 8), 8: ("rkids", np.uint32, 8), 9: ("rvals", np.uint32, 1), 10: ("redges", np.uint32, 8),
                11: ("rstats", np.uint64, 1),   # retained tree: {flattens, in-place patches, garbage child entries, dead nodes, hash entries, image valid}
                12: ("cfilter", np.uint32, 1)}
        for which, (name, dt, width) in spec.items():
            ptr, cnt = C.c_void_p(), C.c_uint64(0)
            self._check(self._lib.gm_debug_table(self._h, which, C.byref(ptr), C.byref(cnt)))
            n = int(cnt.value) * width
            if n == 0:
                out[name] = np.zeros((0, width) if width > 1 else 0, dtype=dt)
                continue
            buf = (C.c_uint8 * (n * np.dtype(dt).itemsize)).from_address(ptr.value)
            a = np.frombuffer(buf, dtype=dt).copy()
            out[name] = a.reshape(-1, width) if width > 1 else a
        return out

    def debug_knob(self, name: str, value: int) -> None:
        """Set a kernel-scheduling knob (gm_debug_knob): tuning / A-B measurements only, results never change.

        tests/test_gpu_edges.py holds these to that promise against the oracle: tok_bulk, sorted_rows, tile_chunk (1..1024),
        k2_ctas (0 = default, 1..3), bucket_bits (site bits * 100 + sub bits, sum <= 18), small_graphs, e2e_chunk (>= 1024
        topics per pipelined chunk) and retain_caps (starting size of the retained lookup's scratch, a multiple of 64 that is
        at least 64; the lookup grows it when a batch overflows it)."""
        self._check(self._lib.gm_debug_knob(self._h, name.encode(), int(value)))

    def kernel_ms(self, max_calls: int = 64) -> np.ndarray:
        """[calls, 3] device milliseconds (tokenise, match, deferred) of the last match calls, oldest first.

        Column 0 is k_tokenize + k_bucket_scan + k_bucket_scatter.  Column 1 is k_match_fast plus, in ids mode,
        k_match_expand, which writes the ids: a roofline that counts the id writes among the match's bytes divides
        them by this column, so the expansion's time belongs in it.  Column 2 is k_match_slow."""
        out = np.zeros((max_calls, 3), dtype=np.float32)
        n = C.c_uint32(0)
        self._check(self._lib.gm_kernel_ms_ring(self._h, _vp(out), max_calls, C.byref(n)))
        return out[:int(n.value)]

    def kernel_launches(self) -> int:
        return int(self._lib.gm_kernel_launches(self._h))


def shard_of(topic_or_filter, n_shards: int) -> int:
    b = _b(topic_or_filter)
    return int(N.lib().gm_shard_of(b, len(b), n_shards))
