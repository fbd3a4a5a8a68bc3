"""Python face of the C++ GpuRouter (rmqtt_b200/csrc/router_host.cpp) — the host-side mirror of rmqtt's
`DefaultRouter` (rmqtt/src/router.rs): `add`, `remove`, `matches`, `topics`, `routes` keep the reference's names,
argument meaning and error behaviour (an invalid filter / topic is an error for that call only)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _native as N
from .engine import Engine, GpuMqttError, pack, _b


@dataclass(frozen=True)
class Id:
    """rmqtt::types::Id — equality covers every field (types.rs:1746-1757); `tag` stands for lid/addrs/username/create_time."""
    node_id: int
    client_id: str
    tag: int = 0


@dataclass(frozen=True)
class SubscriptionOptions:
    """rmqtt::types::SubscriptionOptions (types.rs:565-718): V3 { qos, shared_group } | V5 { qos, no_local, id, shared_group }."""
    qos: int = 0
    is_v5: bool = False
    no_local: bool = False
    sub_id: int = 0
    shared_group: str = ""


@dataclass
class SubRelation:
    node_id: int
    topic_filter: str
    client_id: str
    sub_ids: list = field(default_factory=list)
    group: int = 0          # 0, or id of the (filter, shared group) whose member this is: matches_batch returns every member,
                            # matches_batch_shared the chosen one
    online: bool = True     # matches_batch_shared: False when no eligible member of the group was online


class GpuRouter:
    def __init__(self, engine: Engine | None = None):
        self.engine = engine or Engine()
        self._lib = N.lib()
        h = C.c_void_p()
        rc = self._lib.gmr_create(self.engine._h, C.byref(h))
        if rc != N.GM_OK:
            raise GpuMqttError(rc, "gmr_create")
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.gmr_destroy(self._h)
            self._h = None

    def _check(self, rc):
        if rc != N.GM_OK:
            raise GpuMqttError(rc, self._lib.gm_last_error(self.engine._h).decode())

    @staticmethod
    def _id(i: Id):
        c = _b(i.client_id)
        return N.GmId(i.node_id, c, len(c), 0, i.tag)

    def add(self, topic_filter, id: Id, opts: SubscriptionOptions = SubscriptionOptions()):
        f, g = _b(topic_filter), _b(opts.shared_group)
        gid = self._id(id)
        o = N.GmSubOpts(opts.qos, int(opts.is_v5), int(opts.no_local), 0, opts.sub_id, g if g else None, len(g))
        self._check(self._lib.gmr_add(self._h, f, len(f), C.byref(gid), C.byref(o)))

    def remove(self, topic_filter, id: Id) -> bool:
        f = _b(topic_filter)
        gid = self._id(id)
        rm = C.c_int32(0)
        self._check(self._lib.gmr_remove(self._h, f, len(f), C.byref(gid), C.byref(rm)))
        return bool(rm.value)

    def topics(self) -> int:
        return int(self._lib.gmr_topics(self._h))

    def routes(self) -> int:
        return int(self._lib.gmr_routes(self._h))

    def topics_tree(self) -> int:
        return self.engine.stats()["values"]

    def _relation(self, handle: int):
        f, c = C.c_char_p(), C.c_char_p()
        fl, cl = C.c_uint32(0), C.c_uint32(0)
        self._check(self._lib.gmr_relation(self._h, handle, C.byref(f), C.byref(fl), C.byref(c), C.byref(cl)))
        return C.string_at(f, fl.value).decode(), C.string_at(c, cl.value).decode()

    def set_online(self, node_id: int, client_id: str, online: bool):
        """What Router::is_online answers for (node_id, client_id); a client never named here is online."""
        c = _b(client_id)
        self._check(self._lib.gmr_set_online(self._h, node_id, c, len(c), int(bool(online))))

    def group_members(self, group: int):
        """-> (filter, group name, member handles) of a shared group id (the group_cids of SharedGroupType)."""
        f, g = C.c_char_p(), C.c_char_p()
        fl, gl, n = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        self._check(self._lib.gmr_group(self._h, group, C.byref(f), C.byref(fl), C.byref(g), C.byref(gl), None, 0, C.byref(n)))
        hs = np.zeros(max(1, n.value), dtype=np.uint32)
        self._check(self._lib.gmr_group(self._h, group, C.byref(f), C.byref(fl), C.byref(g), C.byref(gl), hs.ctypes.data_as(C.c_void_p), n.value, C.byref(n)))
        return C.string_at(f, fl.value).decode(), C.string_at(g, gl.value).decode(), [int(x) for x in hs[:n.value]]

    def matches_batch_shared(self, topics, publishers=None, seed: int = 0):
        """Router::matches for a batch with ONE member chosen per matched (filter, shared group), on the device: the draw of
        include/gpumqtt.h gm_relations_choose_device, reproducible from `seed`."""
        return self.matches_batch(topics, publishers, seed=seed)

    def matches_batch(self, topics, publishers=None, *, seed: int | None = None):
        """Router::matches for a batch -> list (per topic) of list[SubRelation], or None for an invalid topic.  Every shared-group
        member is returned unless `seed` is given (see matches_batch_shared)."""
        blob, offs = pack(topics)
        n = len(topics)
        pubs = None
        keep = []
        if publishers is not None:
            arr = (N.GmId * n)()
            for i, p in enumerate(publishers):
                c = _b(p.client_id)
                keep.append(c)
                arr[i] = N.GmId(p.node_id, c, len(c), 0, p.tag)
            pubs = arr
        spans = np.zeros((n, 2), dtype=np.uint32)
        status = np.zeros(n, dtype=np.int32)
        cap_r, cap_s = max(64, 32 * n), max(64, 8 * n)
        while True:
            rels = (N.GmSubRelation * cap_r)()
            sids = np.zeros(cap_s, dtype=np.uint32)
            nr, ns = C.c_uint64(0), C.c_uint64(0)
            args = (pubs, blob.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p), n, spans.ctypes.data_as(C.c_void_p), rels, cap_r,
                    sids.ctypes.data_as(C.c_void_p), cap_s, C.byref(nr), C.byref(ns), status.ctypes.data_as(C.c_void_p))
            if seed is None:
                rc = self._lib.gmr_matches_batch(self._h, *args)
            else:
                rc = self._lib.gmr_matches_batch_shared(self._h, seed, *args)
            if rc == N.GM_ERR_CAPACITY:
                cap_r, cap_s = int(nr.value) + 16, int(ns.value) + 16
                continue
            self._check(rc)
            break
        out = []
        for i in range(n):
            if status[i] != 0:
                out.append(None)
                continue
            lst = []
            for k in range(int(spans[i, 0]), int(spans[i, 0] + spans[i, 1])):
                r = rels[k]
                f, c = self._relation(r.handle)
                lst.append(SubRelation(int(r.node_id), f, c, sids[r.sub_ids_off:r.sub_ids_off + r.sub_ids_cnt].tolist(),
                                       int(r.group) & ~N.GM_SUBREL_OFFLINE, not (int(r.group) & N.GM_SUBREL_OFFLINE)))
            out.append(lst)
        return out

    # ---- secondary readers (router.rs:139-158, 522-546): unique matched filters through the engine's descriptor mode ----
    def matched_filters_batch(self, topics):
        """-> per topic the sorted list of unique matched filter strings, or None for an invalid topic."""
        blob, offs = pack(topics)
        n = len(topics)
        spans = np.zeros((n, 2), dtype=np.uint32)
        status = np.zeros(n, dtype=np.int32)
        cap = max(64, 8 * n)
        while True:
            fl = np.zeros(cap, dtype=np.uint32)
            need = C.c_uint64(0)
            rc = self._lib.gmr_matched_filters_batch(self._h, blob.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p), n, spans.ctypes.data_as(C.c_void_p),
                                                     fl.ctypes.data_as(C.c_void_p), cap, C.byref(need), status.ctypes.data_as(C.c_void_p))
            if rc == N.GM_ERR_CAPACITY:
                cap = int(need.value) + 16
                continue
            self._check(rc)
            break
        out = []
        for i in range(n):
            out.append(None if status[i] != 0 else [int(x) for x in fl[int(spans[i, 0]):int(spans[i, 0] + spans[i, 1])]])
        return out

    def _filter(self, idx: int):
        f, fl, nn = C.c_char_p(), C.c_uint32(0), C.c_uint32(0)
        nodes = np.zeros(64, dtype=np.uint64)
        self._check(self._lib.gmr_filter(self._h, idx, C.byref(f), C.byref(fl), nodes.ctypes.data_as(C.c_void_p), 64, C.byref(nn)))
        return C.string_at(f, fl.value).decode(), [int(x) for x in nodes[:min(64, nn.value)]]

    def has_matches(self, topic):
        """DefaultRouter::_has_matches (router.rs:139-142)."""
        m = self.matched_filters_batch([topic])[0]
        return None if m is None else len(m) > 0

    def get_routes(self, topic, node_id: int):
        """DefaultRouter::_get_routes (router.rs:145-158): Route{this node, filter} per unique matched filter."""
        m = self.matched_filters_batch([topic])[0]
        return None if m is None else sorted((node_id, self._filter(i)[0]) for i in m)

    def get(self, topic):
        """Router::get (router.rs:522-546): Route{node, filter} per unique matched filter and distinct node id among its relations."""
        m = self.matched_filters_batch([topic])[0]
        if m is None:
            return None
        out = []
        for i in m:
            f, nodes = self._filter(i)
            out += [(nid, f) for nid in nodes]
        return sorted(out)

    def matches(self, id: Id, topic):
        return self.matches_batch([topic], [id])[0]
