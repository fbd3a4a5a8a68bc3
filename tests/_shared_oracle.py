"""Restatements used by the shared-subscription tests (test_shared_choice_cpu.py, test_gpu_shared_choice.py).

* `share_key`: the draw's key of include/gpumqtt.h gm_share_key, restated in Python.
* `choose`: the choice among one group's members (the eligible online member with the smallest (key, client_key), else the
  smallest eligible member, flagged offline).
* `SharedRouter`: DefaultRouter::_matches (rmqtt/src/router.rs:162-248) with SharedSubscription::choice (rmqtt/src/subscribe.rs:66-104)
  replaced by that seeded draw, and the group ids / client keys numbered as gpumqtt.h documents.  The filters live in the
  oracle's TopicTree, which returns a filter's value once per visit, so a filter node matched twice gets two choices.

Canonical lines per topic, sorted:
  "3|node|filter|client"                  v3 relation
  "5|node|client|id,id,..."               v5 relation after per-client de-dup (chosen v5 members merged in), ids sorted
  "s|node|filter|group|client|online"     a chosen v3 member of a shared group (online 1 / 0)
"""
from __future__ import annotations

from collections import Counter

from oracle import oracle as orc

M64 = (1 << 64) - 1
NONE = 0xFFFFFFFF


def mix(x: int) -> int:
    x &= M64
    x ^= x >> 30
    x = (x * 0xbf58476d1ce4e5b9) & M64
    x ^= x >> 27
    x = (x * 0x94d049bb133111eb) & M64
    x ^= x >> 31
    return x


def share_key(seed: int, row: int, group: int, occ: int, client_key: int) -> int:
    return mix(mix(seed ^ ((row << 32) | group)) ^ ((occ << 32) | client_key))


def choose(cands, seed, row, group, occ):
    """cands: iterable of (client_key, online, payload) of the ELIGIBLE members -> (payload, online) or None."""
    best = None
    for ck, online, payload in cands:
        k = (0 if online else 1, share_key(seed, row, group, occ, ck), ck)
        if best is None or k < best[0]:
            best = (k, payload)
    return None if best is None else (best[1], best[0][0] == 0)


class SharedRouter:
    """The router-level restatement with the seeded choice."""

    def __init__(self):
        self.tree = orc.TopicTree()
        self.filters: list[str] = []               # filter index (TopicTree value) -> string
        self.filter_idx: dict[str, int] = {}
        self.rel: dict[str, dict[str, tuple]] = {}   # filter -> client -> (node_id, tag, is_v5, no_local, sub_id, group)
        self.group_ids: dict[tuple, int] = {}
        self.client_keys: dict[tuple, int] = {}
        self.offline: set[int] = set()

    def _ck(self, node_id, client):
        return self.client_keys.setdefault((node_id, client), len(self.client_keys))

    def add(self, filt, node_id, client, tag=0, is_v5=False, no_local=False, sub_id=0, group="") -> bool:
        if orc.topic_parse(filt) is None:
            return False
        if filt not in self.filter_idx:
            self.filter_idx[filt] = len(self.filters)
            self.filters.append(filt)
        if filt not in self.rel:
            self.rel[filt] = {}
            self.tree.insert(filt, self.filter_idx[filt])
        self.rel[filt][client] = (node_id, tag, is_v5, no_local, sub_id, group)
        self._ck(node_id, client)
        if group:
            self.group_ids.setdefault((filt, group), len(self.group_ids) + 1)
        return True

    def remove(self, filt, node_id, client, tag=0) -> bool:
        r = self.rel.get(filt, {}).get(client)
        if r is None or (r[0], r[1]) != (node_id, tag):
            return False
        del self.rel[filt][client]
        if not self.rel[filt]:
            del self.rel[filt]
            self.tree.remove(filt, self.filter_idx[filt])
        return True

    def set_online(self, node_id, client, online: bool):
        k = self._ck(node_id, client)
        (self.offline.discard if online else self.offline.add)(k)

    def matches(self, topic, row, seed, pub=None):
        """pub = (node_id, client, tag) of the publisher or None -> canonical lines, or None for an invalid topic."""
        vals = self.tree.matches(topic)
        if vals is None:
            return None
        lines, v5 = [], {}
        for fi, m in sorted(Counter(vals).items()):
            filt = self.filters[fi]
            for occ in range(m):
                groups = {}
                for client, (node, tag, is_v5, no_local, sub_id, group) in self.rel.get(filt, {}).items():
                    if is_v5 and no_local and pub is not None and pub == (node, client, tag):
                        continue                                    # router.rs:184-189
                    if group:
                        groups.setdefault(group, []).append((client, node, is_v5, sub_id))
                    elif is_v5:
                        ids = v5.setdefault((node, client), [])
                        if sub_id:
                            ids.append(sub_id)
                    else:
                        lines.append(f"3|{node}|{filt}|{client}")
                for group, members in groups.items():
                    gid = self.group_ids[(filt, group)]
                    ch = choose(((self._ck(node, client), self._ck(node, client) not in self.offline, (client, node, is_v5, sub_id))
                                 for client, node, is_v5, sub_id in members), seed, row, gid, occ)
                    (client, node, is_v5, sub_id), online = ch
                    if is_v5:
                        ids = v5.setdefault((node, client), [])
                        if sub_id:
                            ids.append(sub_id)
                    else:
                        lines.append(f"s|{node}|{filt}|{group}|{client}|{int(online)}")
        for (node, client), ids in v5.items():
            lines.append(f"5|{node}|{client}|" + ",".join(str(i) for i in sorted(ids)))
        return sorted(lines)
