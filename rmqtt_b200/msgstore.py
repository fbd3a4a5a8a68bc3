"""Python face of the message store (gm_msgstore_*, include/gpumqtt.h): rmqtt-message-storage's RAM backend over an engine
of its own, with the per-client "already forwarded" marks kept, checked and set on the device.

Client ids and (topic filter, shared group) pairs are interned into the keys the C ABI takes: equal pairs get equal keys.
Times are ms since the Unix epoch (rmqtt's timestamp_millis).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N
from .engine import Engine, GpuMqttError, MatchResult, _b, _vp, pack

NO_SHARE = N.GM_MSGSTORE_NO_SHARE


class GpuMessageStore:
    def __init__(self, engine: Engine, initial_mark_slots: int = 0):
        """`engine` is the store's own: the store owns its retained tree.  Give it a max_levels one above the broker's."""
        self._lib = N.lib()
        self.engine = engine
        cfg = N.GmMsgstoreConfig(C.sizeof(N.GmMsgstoreConfig), int(initial_mark_slots))
        h = C.c_void_p()
        rc = self._lib.gm_msgstore_create(engine._h, C.byref(cfg), C.byref(h))
        if rc != N.GM_OK:
            raise GpuMqttError(rc, self._lib.gm_last_error(None).decode())
        self._h = h
        self._clients: dict[bytes, int] = {}
        self._shares: dict[tuple[bytes, bytes], int] = {}

    def close(self):
        if getattr(self, "_h", None):
            self._lib.gm_msgstore_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != N.GM_OK:
            raise GpuMqttError(rc, self._lib.gm_last_error(None).decode())

    # ---- interning -------------------------------------------------------------------------------------------------------
    def client_key(self, client_id) -> int:
        return self._clients.setdefault(_b(client_id), len(self._clients))

    def share_key(self, topic_filter, group) -> int:
        """the key of a shared subscription's (topic filter, group); None for a group of None"""
        if group is None:
            return NO_SHARE
        return self._shares.setdefault((_b(topic_filter), _b(group)), len(self._shares))

    def _mark_keys(self, forwarded):
        """[(client id, None | (topic filter, group))] -> (client keys, share keys)"""
        cl = np.array([self.client_key(c) for c, _ in forwarded], np.uint32)
        sh = np.array([NO_SHARE if s is None else self.share_key(*s) for _, s in forwarded], np.uint32)
        return cl, sh

    # ---- the store -------------------------------------------------------------------------------------------------------
    def store(self, topic, handle: int, expiry_time_at: int, forwarded=()):
        """_set: keep message `handle` until expiry_time_at, already forwarded to `forwarded` ([(client id, None | (filter, group))])"""
        b = _b(topic)
        cl, sh = self._mark_keys(list(forwarded))
        self._check(self._lib.gm_msgstore_store(self._h, b, len(b), int(handle), int(expiry_time_at), _vp(cl), _vp(sh), len(cl)))

    def store_batch(self, topics, handles, expiry_time_at, forwarded=None):
        """n messages at once; forwarded[i] as in store (None: no marks)"""
        blob, offs = pack(topics)
        h = np.ascontiguousarray(handles, np.uint32)
        e = np.ascontiguousarray(expiry_time_at, np.uint64)
        assert len(h) == len(e) == len(offs) - 1
        if forwarded is None:
            self._check(self._lib.gm_msgstore_store_batch(self._h, _vp(blob), _vp(offs), _vp(h), _vp(e), len(h), None, None, None))
            return
        mo = np.zeros(len(h) + 1, np.uint32)
        mo[1:] = np.cumsum([len(f) for f in forwarded])
        cl, sh = self._mark_keys([m for f in forwarded for m in f])
        self._check(self._lib.gm_msgstore_store_batch(self._h, _vp(blob), _vp(offs), _vp(h), _vp(e), len(h), _vp(mo), _vp(cl), _vp(sh)))

    def get_batch_keys(self, now: int, blob: np.ndarray, offs: np.ndarray, clients: np.ndarray, shares: np.ndarray, cap: int | None = None) -> MatchResult:
        """get for a batch of (filter, client key, share key): query i's handles are result.sorted_list(i)"""
        n = len(offs) - 1
        cl = np.ascontiguousarray(clients, np.uint32)
        sh = np.ascontiguousarray(shares, np.uint32)
        assert len(cl) == len(sh) == n
        spans = np.zeros((n, 2), np.uint32)
        status = np.zeros(n, np.int32)
        c = int(cap) if cap is not None else max(1024, 16 * n)
        while True:
            out = np.empty(max(c, 1), np.uint32)
            needed = C.c_uint64(0)
            rc = self._lib.gm_msgstore_get_batch(self._h, int(now), _vp(blob), _vp(offs), n, _vp(cl), _vp(sh), _vp(spans), _vp(out), c,
                                                 C.byref(needed), _vp(status))
            if rc == N.GM_ERR_CAPACITY and cap is None:
                c = int(needed.value)
                continue
            self._check(rc)
            return MatchResult(spans, out[:int(needed.value)], status, int(needed.value))

    def get_batch(self, now: int, filters, clients, shares=None) -> MatchResult:
        """get(client_id, topic_filter, group) for a batch; shares[i] is query i's shared group or None"""
        blob, offs = pack(filters)
        shares = shares if shares is not None else [None] * len(filters)
        cl = np.array([self.client_key(c) for c in clients], np.uint32)
        sh = np.array([self.share_key(f, g) for f, g in zip(filters, shares)], np.uint32)
        return self.get_batch_keys(now, blob, offs, cl, sh)

    def remove_expired(self, now: int, cap: int = 1 << 20) -> np.ndarray:
        """remove_expired_messages: removes up to `cap` messages with expiry_time_at <= now, earliest first -> their handles.
        now = 2**64 - 2 evicts the `cap` earliest-expiring messages (cache_max_count / cache_capacity)."""
        out = np.empty(max(int(cap), 1), np.uint32)
        n = C.c_uint64(0)
        self._check(self._lib.gm_msgstore_remove_expired(self._h, int(now), _vp(out), int(cap), C.byref(n)))
        return out[:int(n.value)].copy()

    def stats(self) -> dict:
        s = N.GmMsgstoreStats()
        self._check(self._lib.gm_msgstore_stats_get(self._h, C.byref(s)))
        return s.as_dict()
