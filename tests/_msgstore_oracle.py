"""rmqtt-message-storage's RAM backend restated with an explicit `now` over the oracle's RetainTree: _set, _get and
remove_expired_messages (rmqtt-plugins/rmqtt-message-storage/src/ram.rs:143-191, 247-367; is_expiry: rmqtt/src/types.rs:1883-1885).
Messages are keyed topic/<msg_id>; forwardeds[msg_id] maps a client to None or its (topic filter, group).  A batch of gets
runs one query at a time, in batch order."""
from __future__ import annotations


class MsgStoreRef:
    def __init__(self, orc):
        self.rt = orc.RetainTree()
        self.topic = {}               # msg_id -> topic
        self.expiry = {}              # msg_id -> expiry_time_at
        self.fwd = {}                 # msg_id -> {client: None | (filter, group)}

    def set(self, topic: str, msg_id: int, expiry_time_at: int, forwarded=()):
        self.rt.insert(f"{topic}/{msg_id}", msg_id)
        self.topic[msg_id] = topic
        self.expiry[msg_id] = expiry_time_at
        d = self.fwd.setdefault(msg_id, {})
        for client, share in forwarded:
            d[client] = share

    def get(self, now: int, client: str, filt: str, group=None):
        """sorted msg ids, None when the filter does not parse"""
        q = filt if (filt == "#" or filt.endswith("/#")) else filt + "/+"
        matched = self.rt.matches(q)
        if matched is None:
            return None
        out = []
        for m in matched:
            d = self.fwd.setdefault(m, {})
            if client in d or (group is not None and any(v == (filt, group) for v in d.values())):
                continue
            if self.expiry[m] < now:
                continue
            d[client] = None if group is None else (filt, group)
            out.append(m)
        return sorted(out)

    def get_batch(self, now: int, filters, clients, groups):
        return [self.get(now, c, f, g) for f, c, g in zip(filters, clients, groups)]

    def remove_expired(self, now: int, limit: int | None = None):
        """removes messages with expiry_time_at <= now, earliest first -> their ids (in removal order)"""
        due = sorted((e, m) for m, e in self.expiry.items() if e <= now)
        if limit is not None:
            due = due[:limit]
        for _, m in due:
            self.rt.remove(f"{self.topic.pop(m)}/{m}")
            del self.expiry[m]
            self.fwd.pop(m, None)
        return [m for _, m in due]

    def evict(self, k: int):
        """the k earliest-expiring messages, whatever their expiry (cache_max_count)"""
        due = sorted((e, m) for m, e in self.expiry.items())[:k]
        for _, m in due:
            self.rt.remove(f"{self.topic.pop(m)}/{m}")
            del self.expiry[m]
            self.fwd.pop(m, None)
        return [m for _, m in due]
