"""Expiry of retained messages as the reference defines it, restated with an explicit `now` over the oracle's RetainTree:
TimedValue (rmqtt/src/types.rs:2275-2296: expired iff now >= deadline), RetainStorage::set_with_timeout, get_message and
remove_expired_messages (rmqtt/src/retain.rs:118-169).  Deadlines are ms since the Unix epoch; 0 = none.  A deadline belongs
to a handle: a value that is replaced or removed loses it, and setting a handle without one clears it."""
from __future__ import annotations

import numpy as np


class TimedRetain:
    def __init__(self, orc):
        self.rt = orc.RetainTree()
        self.val = {}                 # topic -> handle
        self.dl = {}                  # handle -> deadline (non-zero only)

    def set_with_timeout(self, topic: str, h: int, deadline: int = 0):
        old = self.val.get(topic)
        self.rt.insert(topic, h)
        self.val[topic] = h
        if old is not None and old != h:
            self.dl.pop(old, None)
        if deadline:
            self.dl[h] = deadline
        else:
            self.dl.pop(h, None)

    def remove(self, topic: str):
        old = self.val.pop(topic, None)
        self.rt.remove(topic)
        if old is not None:
            self.dl.pop(old, None)
        return old

    def expired(self, h: int, now: int) -> bool:
        d = self.dl.get(h)
        return d is not None and now >= d

    def get_message(self, filt: str, now: int):
        """sorted live handles, None for an invalid filter"""
        r = self.rt.matches(filt)
        return None if r is None else sorted(v for v in r if not self.expired(v, now))

    def match_batch(self, blob, offs, now: int) -> dict:
        """the oracle's match_batch with the expired handles dropped: {"counts", "offsets", "ids"} (ids sorted per filter)"""
        want = self.rt.match_batch(blob, offs)
        counts, o, ids = want["counts"].copy(), want["offsets"], want["ids"]
        keep = []
        for i in range(len(counts)):
            seg = ids[int(o[i]):int(o[i + 1])]
            seg = np.sort(seg[[not self.expired(int(v), now) for v in seg]]) if len(seg) else seg
            if counts[i] >= 0:
                counts[i] = len(seg)
            keep.append(seg.astype(np.uint32))
        no = np.zeros(len(counts) + 1, dtype=np.uint64)
        np.cumsum(np.maximum(counts, 0), out=no[1:])
        return {"counts": counts, "offsets": no, "ids": np.concatenate(keep) if keep else np.zeros(0, np.uint32)}

    def expired_handles(self, now: int):
        return sorted(h for h, d in self.dl.items() if now >= d)

    def remove_expired_messages(self, now: int):
        """removes every expired topic -> their handles, sorted"""
        gone = self.expired_handles(now)
        dead = set(gone)
        for t in [t for t, h in self.val.items() if h in dead]:
            self.remove(t)
        return gone


def seeded_deadlines(topics_values, now: int, rng, share: float = 1.0) -> dict:
    """handle -> deadline for the handles stored under exactly one topic: none, past, exactly `now` and future, in equal parts
    (of a `share` of them)"""
    seen = {}
    for _, v in topics_values:
        seen[v] = seen.get(v, 0) + 1
    out = {}
    for h in sorted(v for v, k in seen.items() if k == 1):
        if rng.random() >= share:
            continue
        kind = rng.randrange(4)
        if kind == 1:
            out[h] = max(1, now - 1 - rng.randrange(1000))
        elif kind == 2:
            out[h] = now
        elif kind == 3:
            out[h] = now + 1 + rng.randrange(1000)
    return out
