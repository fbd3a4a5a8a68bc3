"""Tile-shape corpus of the fast path's id expansion: k_match_fast stores the matched value sets of every tile whose ids fit
(one TileRec per tile, the sets lane-major in the item array) and k_match_expand turns them into ids, 32 sets per step.

Every topic `te/x/p<k>/a/b/c/d/e` matches exactly the value sets its profile dials: set i is the value set of the i-th of the
38 filters `+/+/p<k>/...` that match it, with a chosen number of members (or one chosen value: 0 and 2^32-1 take the
single-value shortcut).  Each case states its F (matched sets) and M (ids); `check_against_oracle` re-derives both one topic
at a time, so the corpus cannot drift away from the shapes it claims.

All valid non-`$` topics share their first two levels, so they share one locality bucket: those rows of a batch are its
tiles in batch order on the emulator (one thread per row, in order) and in some order on the GPU.  Invalid topics sort
into bucket 0, ahead of them; `$` topics into a bucket of their own, whose place in the order the corpus does not know.
A batch of exactly 32 rows of the shared bucket is one tile whatever the order.

Value ranges: corpus values below 2^24, the two bulk sets at 2^24 and 2^25, 0 and 2^32-1; `poison_batch` values from
0x70000000; the output pattern of the tests fills [0x80000000, 0xF0000000), which no match ever yields.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from _edges import CNT_BIG, K2_POOL_ROWS, K2_SMEM_DESCS, SMALL_TIERS, pack_topics
from oracle import oracle as orc

MAX_FAST_SETS = K2_SMEM_DESCS + K2_POOL_ROWS      # 32: more matched sets and k_match_fast defers the topic
PREFIX = "te/x"
LIT = "abcde"
BIG, HUGE = "big", "huge"                          # a 65534-member set (largest in-line) / a 65535-member one (CNT_BIG: deferred)
POISON_BASE = 0x70000000
PATTERN_LO, PATTERN_SPAN = 0x80000000, 0x70000000


def pattern(n: int, salt: int) -> np.ndarray:
    """n position-dependent words in [PATTERN_LO, PATTERN_LO + PATTERN_SPAN): a stray copy of a valid id never equals one."""
    i = np.arange(n, dtype=np.uint64)
    return (PATTERN_LO + (i * np.uint64(0x9E3779B1) + np.uint64(salt * 7919)) % np.uint64(PATTERN_SPAN)).astype(np.uint32)


def set_filters(root: str) -> list[str]:
    """The 38 filters that match `te/x/<root>/a/b/c/d/e`: 32 literal / '+' combinations, then 6 '#' filters."""
    combos = [f"+/+/{root}/" + "/".join("+" if m >> i & 1 else LIT[i] for i in range(5)) for m in range(32)]
    hashes = [f"+/+/{root}/" + "".join(x + "/" for x in LIT[:j]) + "#" for j in range(6)]
    return combos + hashes


@dataclass(frozen=True)
class TCase:
    topic: bytes
    F: int | None            # matched value sets; None: Topic::from_str fails
    M: int                   # matched ids
    deferred: bool = False   # k_match_fast hands the topic to k_match_slow


@dataclass
class TileCorpus:
    adds: list = field(default_factory=list)       # (filter, value)
    bulk: list = field(default_factory=list)       # (filter, first value, number of values)
    trees: dict = field(default_factory=dict)
    batches: dict = field(default_factory=dict)    # name -> [TCase]
    profiles: dict = field(default_factory=dict)   # set specs -> TCase
    next_value: int = 16
    next_poison: int = POISON_BASE

    def profile(self, specs, poison: bool = False) -> TCase:
        """The topic whose matched sets are `specs`: an int k (k fresh values), ("v", x) (the single value x), BIG or HUGE."""
        key = (poison, tuple(specs))
        if key in self.profiles:
            return self.profiles[key]
        root = f"{'z' if poison else 'p'}{len(self.profiles)}"
        assert len(specs) <= 38
        m, deferred = 0, len(specs) > MAX_FAST_SETS
        for f, s in zip(set_filters(root), specs):
            if isinstance(s, int):
                for _ in range(s):
                    if poison:
                        self.adds.append((f, self.next_poison)); self.next_poison += 1
                    else:
                        self.adds.append((f, self.next_value)); self.next_value += 1
                m += s
            elif s in (BIG, HUGE):
                k = CNT_BIG - 1 if s == BIG else CNT_BIG
                self.bulk.append((f, 1 << 24 if s == BIG else 1 << 25, k))
                m += k
                deferred |= s == HUGE
            else:
                self.adds.append((f, s[1]))
                m += 1
        c = self.profiles[key] = TCase(f"{PREFIX}/{root}/a/b/c/d/e".encode(), len(specs), m, deferred)
        return c

    def load_oracle(self) -> orc.TopicTree:
        tree = orc.TopicTree()
        for f, v in self.adds:
            tree.insert(f, v)
        for f, v0, k in self.bulk:
            tree.bulk_insert(*pack_topics([f] * k), np.arange(v0, v0 + k, dtype=np.uint32))
        return tree

    def load_engine(self, eng):
        for f, v in self.adds:
            eng.add(f, v)
        for f, v0, k in self.bulk:
            eng.bulk_load(*pack_topics([f] * k), np.arange(v0, v0 + k, dtype=np.uint32))

    def packed(self, name: str):
        return pack_topics([c.topic for c in self.batches[name]])

    def n_deferred(self, name: str) -> int:
        return sum(c.deferred for c in self.batches[name])

    def emu_order(self, name: str) -> list[TCase] | None:
        """The rows in the emulator's locality order (invalid rows, then the shared bucket in batch order); None when the
        batch has `$` rows, whose bucket may sort anywhere."""
        cs = self.batches[name]
        if any(c.topic.startswith(b"$") for c in cs):
            return None
        return [c for c in cs if c.F is None] + [c for c in cs if c.F is not None]

    def tiles(self, name: str) -> list[int] | None:
        """Value sets the item array holds per tile, rows in the emulator's order (None: not known, see `emu_order`)."""
        rows = self.emu_order(name)
        return None if rows is None else [sum(c.F or 0 for c in rows[i:i + 32] if not c.deferred) for i in range(0, len(rows), 32)]

    def tile_ids(self, name: str) -> list[int] | None:
        """Ids k_match_fast reserves per tile, rows in the emulator's order (None: not known, see `emu_order`)."""
        rows = self.emu_order(name)
        return None if rows is None else [sum(c.M for c in rows[i:i + 32] if not c.deferred) for i in range(0, len(rows), 32)]

    def poison_batch(self, n: int, sets: int = 24, size: int = 3) -> list[TCase]:
        """n rows of `sets` sets of `size` values each, every value from POISON_BASE on: ids that no checked batch yields."""
        return [self.profile([size + (i + j) % 2 for j in range(sets)], poison=True) for i in range(4)] * (n // 4) + \
            [self.profile([size] * sets, poison=True)] * (n % 4)


def _lanes(c: TileCorpus, per_lane):
    return [c.profile(s) if s is not None else NOMATCH for s in per_lane]


NOMATCH = TCase(f"{PREFIX}/none".encode(), 0, 0)
INVALID = TCase(f"{PREFIX}/a+b".encode(), None, 0)
DOLLAR = TCase(f"${PREFIX}/p0/a/b/c/d/e".encode(), 0, 0)


def tile_corpus() -> TileCorpus:
    c = TileCorpus()
    add = c.adds.append
    # a deferred topic by depth: 10 levels in a trie 10 levels deep
    add(("+/+/d/#", 9)); add(("+/+/d/" + "/".join(["+"] * 7), 10))
    deep = TCase(f"{PREFIX}/d/1/2/3/4/5/6/7".encode(), 2, 2, True)
    holes = [NOMATCH, INVALID, DOLLAR, deep, c.profile([1] * (MAX_FAST_SETS + 1)), c.profile([HUGE])]

    def sizes(f, lane):                            # set sizes of a lane with f sets: 1 (single), 2 and 3 in turn
        return [1 + (lane + j) % 3 for j in range(f)]

    mix = [c.profile(s) for s in ([1], [2], [("v", 0)], [("v", 0xFFFFFFFF)], [33], [1, 2, 3], [("v", 0), 2, ("v", 0xFFFFFFFF), 33],
                                  [5] * 9, [1] * 32, [3, 1] * 16, [("v", 0xFFFFFFFF), 1] * 16)]

    # ---- value sets per tile: 31, 32, 33, 64, 65 (one tile each), 1024 (every lane at 32 sets); a batch whose every row has 32
    #      sets fills the item array (32 per row) exactly
    for t in (31, 32, 33, 64, 65):
        c.batches[f"items{t}"] = _lanes(c, [sizes(t // 32 + (i < t % 32), i) or None for i in range(32)])
    c.batches["items1024"] = [c.profile(sizes(32, i % 4)) for i in range(32)]
    c.batches["full32"] = [c.profile(sizes(32, i % 4)) for i in range(70)]
    # ---- ids in one 32-set step: 31, 32, 33, 63; one step with the 65534-member set among single values
    singles = [[("v", 0)], [("v", 0xFFFFFFFF)], [1]]
    c.batches["step31"] = _lanes(c, [singles[i % 3] for i in range(31)] + [None])
    c.batches["step32"] = _lanes(c, [singles[i % 3] for i in range(32)])
    c.batches["step33"] = _lanes(c, [singles[i % 3] for i in range(31)] + [[2]])
    c.batches["step63"] = _lanes(c, [singles[i % 3] for i in range(31)] + [[32]])
    c.batches["step_big"] = _lanes(c, [singles[i % 3] for i in range(5)] + [[BIG]] + [singles[i % 3] for i in range(26)])
    # ---- single values 0 / 2^32-1 and 2- / 33-member sets, lane by lane and inside one lane
    alt = [[("v", 0)], [2], [("v", 0xFFFFFFFF)], [33], [("v", 0), 2, ("v", 0xFFFFFFFF), 33], [33, ("v", 0), 2, ("v", 0xFFFFFFFF)] * 4]
    c.batches["singles"] = _lanes(c, [alt[i % len(alt)] for i in range(64)])
    # ---- lanes without ids at 0, 15 and 31 of every tile, one kind per tile, all rows in the shared bucket: no match and the
    #      three kinds of deferred topic (on the emulator exactly those lanes; on the GPU somewhere in the tile)
    kept = [h for h in holes if h not in (INVALID, DOLLAR)]
    c.batches["holes"] = [kept[t] if i in (0, 15, 31) else mix[(t * 32 + i) % len(mix)] for t in range(len(kept)) for i in range(32)]
    # ---- invalid and `$` rows among the others: they sort out of the shared bucket (invalid rows ahead of it, at the first
    #      lanes of the first tile on the emulator; `$` rows into a bucket of their own), so the shared bucket's rows move up
    c.batches["holes_sorted_out"] = [(INVALID, DOLLAR)[t] if i in (0, 15, 31) else mix[(t * 32 + i) % len(mix)] for t in range(2) for i in range(32)]
    # ---- partial last tiles, and the small-graph tiers at their capacities and far below them
    pool = [(holes[-1] if i == 60 else holes[(i // 11) % (len(holes) - 1)]) if i % 11 == 5 else mix[(i * 7) % len(mix)] for i in range(2049)]
    for n in (1, 31, 33, 63, 65, 2049):
        c.batches[f"p{n}"] = pool[:n]
    light = [x for x in pool if x.M < 40 and x not in holes[-2:]]
    for (cap_n, cap_blob, cap_out), tier in zip(SMALL_TIERS, (0, 1)):
        for name, n in ((f"g{tier}_at", cap_n), (f"g{tier}_low", 3 if tier == 0 else 100)):
            rows = c.batches[name] = [light[(i * 5) % len(light)] for i in range(n)]
            assert sum(x.M for x in rows) <= cap_out and len(b"".join(x.topic for x in rows)) <= cap_blob
    # ---- poison batches: as many rows as a small-graph tier's capacity (the same scratch layout as that tier's graph), and
    #      more; their ids come from values no other batch yields
    for n in (64, 2048, 4096):
        c.batches[f"z{n}"] = c.poison_batch(n)
    # ... and poison batches that themselves run as each small-graph tier's graph (within its text and output capacities)
    for (cap_n, cap_blob, cap_out), tier in zip(SMALL_TIERS, (0, 1)):
        rows = c.batches[f"z{tier}_graph"] = c.poison_batch(cap_n, sets=16)
        assert sum(x.M for x in rows) <= cap_out and len(b"".join(x.topic for x in rows)) <= cap_blob
    return c


SHAPES = ["items31", "items32", "items33", "items64", "items65", "items1024", "full32", "step31", "step32", "step33", "step63", "step_big",
          "singles", "holes", "holes_sorted_out", "p1", "p31", "p33", "p63", "p65", "p2049", "g0_at", "g0_low", "g1_at", "g1_low"]


def check_against_oracle(c: TileCorpus, tree: orc.TopicTree | None = None):
    """Every distinct topic: F, M and validity as the case states; and the tile shapes the corpus claims to reach."""
    tree = tree or c.load_oracle()
    seen = set()
    for cases in c.batches.values():
        for x in cases:
            if x in seen:
                continue
            seen.add(x)
            want = tree.match_batch(*pack_topics([x.topic]), want_ids=False)
            if x.F is None:
                assert want["counts"][0] < 0, x.topic
            else:
                assert (int(want["counts"][0]), want["counters"]["F"]) == (x.M, x.F), (x.topic, want["counts"][0], want["counters"]["F"], x.M, x.F)
    for t in (31, 32, 33, 64, 65, 1024):
        assert c.tiles(f"items{t}") == [t]
    assert c.tiles("full32") == [1024, 1024, 192]
    assert [sum(x.M for x in c.batches[f"step{k}"]) for k in (31, 32, 33, 63)] == [31, 32, 33, 63]
