"""A deterministic writer script for the flush-concurrency tests, the result every prefix of it must give, and the checker.

The writer mutates only the `w` namespace: every filter, extra-tree filter and retained topic it writes starts with the
level `w`, which the workload generator never produces, so the background's own results never change.  Background
wildcard filters may still match the writer's topics; the expected lists of the probes include them.

A *state* is a prefix of the script's mutations: state p is the content after the first p of them.  A reader that took
`Progress.before()` right before a call and `Progress.after()` once its result was on the host must get the result of ONE
legal state p with lo <= p <= hi (`window`).  With automatic flushes every prefix is legal (a reader's implicit flush can
ship a step half-done); with GM_FLAG_MANUAL_FLUSH only the prefixes the writer flushed are.

The expected result of a probe at state p is its static background list plus the values of the live writer entries that
match it.  Which writer entries can match a probe is computed once with the oracle; `Model` then replays the script over
those sets and keeps, per probe, the list of versions (first state, sorted list) instead of querying the oracle for every
prefix and probe."""
from __future__ import annotations

import bisect
from collections import Counter

import numpy as np

from oracle import oracle as orc
from rmqtt_b200 import workload as wl
from rmqtt_b200.engine import pack

K, W = 2000, 300                  # steps; a step's entries are removed W steps later
NOW = 1_700_000_000_000           # the lookups' clock (ms since the Unix epoch), fixed and in the past
LATE = 1 << 62                    # any clock after every deadline of the script (the wall clock of the batchers' lookups)
VBASE = 1 << 20                   # values and retained handles of step i: VBASE + i (the background uses 0 .. 7999)
DEEP = "w/a/b/c/d/e/f/g/h/i/j/k"  # 12 levels: max_depth passes 8 while it is subscribed
DEEP_ADD, DEEP_REMOVE, COMPACT_AT, TREE_FROM, DEADLINE_FROM = 300, 700, 1500, 200, K // 4
N_BG_SUBS, N_BG_TOPICS, N_BG_RETAINED, N_BG_FILTERS = 8000, 20000, 5000, 3000

SUB_PROBES = ["w/x", DEEP, DEEP + "/l"] + [f"w/{j}/y" for j in range(0, K, 50)] + [f"w/{'L' * 30}{i}/y" for i in range(50, K, 200)]
TREE_PROBES = ["w/x"] + [f"w/{j}/y" for j in range(TREE_FROM, K, 100)]          # rows on extra tree 1
RET_PROBES = ["w/#", "w/+", "+/+", "w/+/#"] + [f"w/{j}" for j in range(0, K, 53)]   # (53: every kind of deadline)
RET_BIG_PROBES = ["#"]            # matches the whole background too: too many handles for the smallest lookup graph
INVALID_TOPICS = ["w/#/x", "w/a+"]
INVALID_FILTERS = ["w/#/x", "w/a+"]


def _long_level(i: int) -> str:
    return "L" * 30 + str(i)          # longer than 27 bytes: the level goes to the string pool and dict_lookup_long


def deadline(i: int) -> int:
    """The deadline of step i's retained message: none before DEADLINE_FROM, then none / before / at / after NOW in turn."""
    if i < DEADLINE_FROM:
        return 0
    return (0, NOW - 1 - i % 500, NOW, NOW + 1 + i)[i % 4]


def script():
    """-> ops: ("add" | "rm", tree, filter, value), ("rset", topic, handle, deadline), ("rrm", topic), ("compact",), ("flush",)"""
    ops = []
    for i in range(K):
        v = VBASE + i
        ops += [("add", 0, f"w/{i}/+", v), ("add", 0, "w/#", v)]
        if i >= W:
            ops += [("rm", 0, f"w/{i - W}/+", v - W), ("rm", 0, "w/#", v - W)]
        if i % 100 == 50:
            ops.append(("add", 0, f"w/{_long_level(i)}/+", v))
        if i == DEEP_ADD:
            ops.append(("add", 0, DEEP, v))
        if i == DEEP_REMOVE:
            ops.append(("rm", 0, DEEP, VBASE + DEEP_ADD))
        if i >= TREE_FROM and i % 10 == 0:          # extra tree 1 is created at TREE_FROM
            ops.append(("add", 1, "w/+/#", v))
        ops.append(("rset", f"w/{i}", v, deadline(i)))
        if i >= W:
            ops.append(("rrm", f"w/{i - W}"))
        if i == COMPACT_AT:                          # after the step's mutations: it flushes, so it ships a step boundary
            ops.append(("compact",))
        ops.append(("flush",))
    return ops


def is_mutation(op) -> bool:
    return op[0] not in ("flush", "compact")


def apply(eng, op):
    k = op[0]
    if k == "add":
        eng.add_tree(op[1], op[2], op[3]) if op[1] else eng.add(op[2], op[3])
    elif k == "rm":
        eng.remove_tree(op[1], op[2], op[3]) if op[1] else eng.remove(op[2], op[3])
    elif k == "rset":
        eng.retain_set(op[1], op[2], op[3] or None)
    elif k == "rrm":
        eng.retain_remove(op[1])
    elif k == "compact":
        eng.compact()
    else:
        eng.flush()


class Progress:
    """The writer's counters.  Each is written by the writer thread only and only grows."""

    def __init__(self):
        self.mut_started = self.mut_done = 0        # mutations begun / finished
        self.flush_started = self.flush_done = 0    # the state the last flush begun / finished ships
        self.flushes_started = self.flushes_done = 0

    def before(self):
        return (self.mut_done, self.flush_done, self.flushes_done)

    def after(self):
        return (self.mut_started, self.flush_started, self.flushes_started)


def window(before, after, manual: bool):
    """[lo, hi] of the states a call bracketed by `before` / `after` may show"""
    return (before[1], after[1]) if manual else (before[0], after[0])


def spans_flush(before, after) -> bool:
    return after[2] > before[2]


def run_writer(eng, ops, prog: Progress, on_flush=None):
    for op in ops:
        if is_mutation(op):
            prog.mut_started += 1
            apply(eng, op)
            prog.mut_done += 1
        else:
            prog.flush_started = prog.mut_done
            prog.flushes_started += 1
            apply(eng, op)
            prog.flush_done = prog.flush_started
            prog.flushes_done += 1
            if on_flush:
                on_flush()


def _s(b) -> str:
    return b.decode() if isinstance(b, (bytes, bytearray)) else b


class Background:
    """The seeded background: C2-scaled subscriptions and publish topics, C4 retained topics and SUBSCRIBE filters, with
    their oracle results (which the writer never changes)."""

    def __init__(self):
        cfg = wl.C2.scaled(n_subs=N_BG_SUBS, n_topics=N_BG_TOPICS)
        self.subs = wl.gen_subs(cfg)
        self.topics = [_s(t) for t in wl.unpack(*wl.gen_topics(cfg))]
        self.retained = wl.gen_retained(wl.C4, N_BG_RETAINED)
        self.filters = [_s(f) for f in wl.unpack(*wl.gen_retain_filters(wl.C4, N_BG_FILTERS))]
        for s in [_s(x) for x in wl.unpack(*self.subs[:2])] + self.topics + [_s(x) for x in wl.unpack(*self.retained[:2])] + self.filters:
            assert s.split("/")[0] != "w", s
        self.tree, self.rtree = orc.TopicTree(), orc.RetainTree()
        self.tree.bulk_insert(*self.subs)
        self.rtree.bulk_insert(*self.retained)
        self.topic_want = _lists(self.tree.match_batch(*pack(self.topics)))
        self.filter_want = _lists(self.rtree.match_batch(*pack(self.filters)))

    def load(self, eng):
        eng.bulk_load(*self.subs)
        eng.retain_bulk_load(*self.retained)
        eng.flush()


def _lists(want):
    o, ids = want["offsets"], want["ids"]
    return [tuple(sorted(ids[int(o[i]):int(o[i + 1])].tolist())) if want["counts"][i] >= 0 else None for i in range(len(want["counts"]))]


class Model:
    """Expected results of every state of `ops` for the probe keys ("sub", tree, topic) and ("ret", now, filter)."""

    def __init__(self, ops, bg: Background):
        muts = [op for op in ops if is_mutation(op)]
        self.n = len(muts)
        self.flushed = np.zeros(self.n + 1, dtype=bool)     # the states a flush shipped (state 0: the loaded background)
        self.flushed[0] = True
        p = 0
        for op in ops:
            if is_mutation(op):
                p += 1
            else:
                self.flushed[p] = True
        self.first_deadline = next(m for m, op in enumerate(muts, 1) if op[0] == "rset" and op[3])
        keys = [("sub", 0, t) for t in SUB_PROBES] + [("sub", 1, t) for t in TREE_PROBES] + \
               [("ret", now, f) for now in (NOW, LATE) for f in RET_PROBES + RET_BIG_PROBES]
        # the writer entries each probe can match, from the oracle: filters per tree, retained topics
        wf = {0: sorted({op[2] for op in muts if op[0] in ("add", "rm") and op[1] == 0}),
              1: sorted({op[2] for op in muts if op[0] in ("add", "rm") and op[1] == 1})}
        wt = sorted({op[1] for op in muts if op[0] in ("rset", "rrm")})
        ftrees = {}
        for tr, fl in wf.items():
            ftrees[tr] = orc.TopicTree()
            for k, f in enumerate(fl):
                ftrees[tr].insert(f, k)
        ttree = orc.RetainTree()
        for k, t in enumerate(wt):
            ttree.insert(t, k)
        by_filter, by_topic = {}, {}                # (tree, filter) / topic -> the keys whose lists it feeds
        static = {}
        for key in keys:
            if key[0] == "sub":
                _, tr, t = key
                for k in ftrees[tr].matches(t):
                    by_filter.setdefault((tr, wf[tr][k]), []).append(key)
                static[key] = bg.tree.matches(t) if tr == 0 else []
            else:
                _, now, f = key
                for k in ttree.matches(f):
                    by_topic.setdefault(wt[k], []).append(key)
                static[key] = bg.rtree.matches(f)
        # the background never changes what a background probe matches (its lists are static)
        for t in bg.topics:
            assert not ftrees[0].matches(t), t
        for f in bg.filters:
            assert not ttree.matches(f), f
        live = {key: Counter() for key in keys}
        self.vstart = {key: [0] for key in keys}
        self.vlist = {key: [tuple(sorted(static[key]))] for key in keys}
        pairs, rstate = set(), {}

        def publish(key, m):
            lst = tuple(sorted(static[key] + list(live[key].elements())))
            if lst != self.vlist[key][-1]:
                self.vstart[key].append(m)
                self.vlist[key].append(lst)

        for m, op in enumerate(muts, 1):
            if op[0] in ("add", "rm"):
                _, tr, f, v = op
                pair = (tr, f, v)
                if (op[0] == "add") == (pair in pairs):       # TopicTree: adding a present or removing an absent pair changes nothing
                    continue
                pairs.add(pair) if op[0] == "add" else pairs.discard(pair)
                for key in by_filter.get((tr, f), ()):
                    live[key][v] += 1 if op[0] == "add" else -1
                    publish(key, m)
            else:
                t = op[1]
                old = rstate.pop(t, None)
                if op[0] == "rset":
                    rstate[t] = (op[2], op[3])
                for key in by_topic.get(t, ()):
                    now = key[1]
                    if old is not None and not (old[1] and now >= old[1]):
                        live[key][old[0]] -= 1
                    if op[0] == "rset" and not (op[3] and now >= op[3]):
                        live[key][op[2]] += 1
                    publish(key, m)

    def expected(self, key, p: int):
        return self.vlist[key][bisect.bisect_right(self.vstart[key], p) - 1]

    def states(self, gots: dict, lo: int, hi: int, manual: bool) -> np.ndarray:
        """The legal states in [lo, hi] whose expected list equals got for every (key -> got) of `gots`."""
        lo, hi = max(lo, 0), min(hi, self.n)
        if hi < lo:
            return np.zeros(0, dtype=np.int64)
        ok = self.flushed[lo:hi + 1].copy() if manual else np.ones(hi - lo + 1, dtype=bool)
        for key, got in gots.items():
            st, ls = self.vstart[key], self.vlist[key]
            m = np.zeros_like(ok)
            v = bisect.bisect_right(st, lo) - 1
            while v < len(st) and st[v] <= hi:
                if ls[v] == got:
                    end = st[v + 1] - 1 if v + 1 < len(st) else self.n
                    m[max(st[v], lo) - lo:min(end, hi) - lo + 1] = True
                v += 1
            ok &= m
            if not ok.any():
                break
        return lo + np.nonzero(ok)[0]


class Batch:
    """One reader's batch.  rows: (text, tree, spec) with spec a probe key, None (an invalid topic or filter: status -2) or
    the static sorted list of a background row."""

    def __init__(self, rows):
        self.rows = rows
        self.texts = [r[0] for r in rows]
        self.trees = np.asarray([r[1] for r in rows], dtype=np.uint32)
        self.blob, self.offs = pack(self.texts)
        is_key = lambda spec: len(spec) == 3 and spec[0] in ("sub", "ret")
        self.probes = [(i, r[2]) for i, r in enumerate(rows) if r[2] is not None and is_key(r[2])]
        self.invalid = np.asarray([i for i, r in enumerate(rows) if r[2] is None], dtype=np.int64)
        bg = [i for i, r in enumerate(rows) if r[2] is not None and not is_key(r[2])]
        self.bg = np.asarray(bg, dtype=np.int64)
        self.bg_counts = np.asarray([len(rows[i][2]) for i in bg], dtype=np.int64)
        self.bg_ids = np.asarray([v for i in bg for v in rows[i][2]], dtype=np.uint32)


def check(model: Model, batch: Batch, status, counts, ids, lo: int, hi: int, manual: bool) -> np.ndarray:
    """Checks one call's result (status int32[n], counts int64[n], ids uint32[] sorted within each row, rows in order) ->
    the states it is consistent with; AssertionError when it is consistent with none."""
    status, counts = np.asarray(status), np.asarray(counts, dtype=np.int64)
    n = len(batch.rows)
    assert len(status) == n and len(counts) == n
    assert (status[batch.invalid] == -2).all(), f"invalid rows got status {status[batch.invalid].tolist()}"
    valid = status == 0
    bad = np.nonzero(~valid)[0]
    assert set(bad.tolist()) == set(batch.invalid.tolist()), f"rows {sorted(set(bad.tolist()) - set(batch.invalid.tolist()))[:5]} failed"
    cnt = np.where(valid, counts, 0)
    starts = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(cnt, out=starts[1:])
    assert len(ids) == starts[-1], (len(ids), int(starts[-1]))
    got_bg = counts[batch.bg]
    if not (got_bg == batch.bg_counts).all():
        i = int(batch.bg[np.nonzero(got_bg != batch.bg_counts)[0][0]])
        raise AssertionError(f"background row {batch.texts[i]!r}: {ids[starts[i]:starts[i + 1]].tolist()} != {list(batch.rows[i][2])}")
    is_bg = np.zeros(n, dtype=bool)
    is_bg[batch.bg] = True
    bg_ids = ids[np.repeat(is_bg, cnt)]
    if not (bg_ids == batch.bg_ids).all():
        raise AssertionError("a background row's list differs from its static oracle list")
    gots = {}
    for i, key in batch.probes:
        got = tuple(ids[starts[i]:starts[i + 1]].tolist())
        if gots.setdefault(key, got) != got:
            raise AssertionError(f"two rows of {key} differ within one call")
    st = model.states(gots, lo, hi, manual)
    if len(st) == 0:
        raise AssertionError(f"no legal state in [{lo}, {hi}] gives this result: " + describe(model, gots, lo, hi, manual))
    return st


def describe(model: Model, gots: dict, lo: int, hi: int, manual: bool) -> str:
    """Which states each probe alone is consistent with (for the failure message)"""
    parts = []
    for key, got in gots.items():
        alone = model.states({key: got}, 0, model.n, manual)
        inside = alone[(alone >= lo) & (alone <= hi)]
        parts.append(f"{key}: {len(got)} ids, states {alone[:3].tolist()}..{alone[-3:].tolist()} ({len(inside)} in the window)")
    return "; ".join(parts[:12])


def canonical_lists(spans, ids, status):
    """(status, counts, ids sorted within each row) of a result given as spans (offset, count) into ids"""
    spans = np.asarray(spans).reshape(-1, 2).astype(np.int64)
    status = np.asarray(status).astype(np.int32)
    counts = np.where(status == 0, spans[:, 1], -1)
    pos = np.maximum(counts, 0)
    total = int(pos.sum())
    if total == 0:
        return status, counts, np.zeros(0, dtype=np.uint32)
    seg = np.repeat(np.arange(len(counts)), pos)
    starts = np.zeros(len(counts) + 1, dtype=np.int64)
    np.cumsum(pos, out=starts[1:])
    src = np.repeat(spans[:, 0], pos) + np.arange(total) - np.repeat(starts[:-1], pos)
    vals = np.asarray(ids).astype(np.uint32)[src]
    return status, counts, vals[np.lexsort((vals, seg))]
