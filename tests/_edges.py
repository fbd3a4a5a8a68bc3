"""Boundary corpus of the match kernels: one subscription trie, the batches that exercise it, and a small retained tree.

Every case reaches its boundary by construction and states what it expects: for every topic the number of matched filter
nodes F (None: Topic::from_str fails) and whether k_match_fast must hand it to the deferred kernel.  `check_against_oracle`
re-derives F from the oracle one topic at a time, so the corpus cannot drift away from the boundaries it claims to hit.

The constants mirror rmqtt_b200/csrc (kernels.cuh, layout.h, pipeline.cuh); the tests assert the byte counts that depend on them.
"""
from __future__ import annotations

import random
from dataclasses import dataclass, field

import numpy as np

from oracle import oracle as orc

K2_SMEM_DESCS = 8            # matched value sets per topic in shared memory (kernels.cuh)
K2_POOL_ROWS = 24            # ... plus the spill rows in global memory before the topic is deferred (pipeline.cuh)
K2_FAST_L = 8                # levels k_match_fast walks; deeper topics are deferred
CNT_BIG = 0xFFFF             # a value set of >= 65535 members goes through `ranges` (deferred kernel only)
DICT_INLINE_MAX = 27         # level strings up to 27 bytes live in the dictionary slot, longer ones in the pool
WIDE_FANOUT = 48             # more literal children than this: the node's edges go into the child filter
TOK_THREADS = 256            # topics per k_tokenize CTA
TOK_STAGE_BYTES = 24 * 1024  # the bulk tokeniser stages at most this much text per CTA
SMALL_TIERS = ((64, 8 * 1024, 4096), (2048, 192 * 1024, 128 * 1024))   # small-batch graphs: (topics, text bytes, output elements)

# Root wildcards: every valid topic outside a `$` root matches both.  Their values are the extremes of u32.
ROOT_WILD = (("#", 0xFFFFFFFF), ("+/#", 0))
W = len(ROOT_WILD)


@dataclass
class Case:
    topic: bytes
    F: int | None            # matched filter nodes; None = invalid topic
    big: bool = False        # matches a value set of >= 65535 members


@dataclass
class Corpus:
    adds: list = field(default_factory=list)        # (filter, value)
    bulk: list = field(default_factory=list)        # (filter, first value, number of values): one value set per filter
    trees: dict = field(default_factory=dict)       # extra tree id -> [(filter, value)]
    batches: dict = field(default_factory=dict)     # name -> [Case]
    max_depth: int = 0

    def levels(self, topic: bytes) -> int:
        return topic.count(b"/") + 1

    def deferred(self, c: Case) -> bool:
        """k_match_fast defers a valid topic with more than K2_FAST_L levels to walk, a huge value set, or more matched sets
        than shared memory plus the spill pool hold."""
        if c.F is None:
            return False
        return min(self.levels(c.topic), self.max_depth) > K2_FAST_L or c.big or c.F > K2_SMEM_DESCS + K2_POOL_ROWS

    def n_deferred(self, name: str) -> int:
        return sum(self.deferred(c) for c in self.batches[name])

    def packed(self, name: str):
        return pack_topics([c.topic for c in self.batches[name]])

    def load_oracle(self) -> orc.TopicTree:
        tree = orc.TopicTree()
        for f, v in self.adds:
            tree.insert(f, v)
        for f, v0, k in self.bulk:
            tree.bulk_insert(*pack_topics([f] * k), np.arange(v0, v0 + k, dtype=np.uint32))
        return tree

    def load_engine(self, eng):
        """Into an rmqtt_b200 Engine (or anything with add / bulk_load / add_tree)."""
        for f, v in self.adds:
            eng.add(f, v)
        for f, v0, k in self.bulk:
            eng.bulk_load(*pack_topics([f] * k), np.arange(v0, v0 + k, dtype=np.uint32))
        for tr, fl in self.trees.items():
            for f, v in fl:
                eng.add_tree(tr, f, v)

    def tree_oracles(self) -> dict:
        out = {0: self.load_oracle()}
        for tr, fl in self.trees.items():
            t = orc.TopicTree()
            for f, v in fl:
                t.insert(f, v)
            out[tr] = t
        return out


def pack_topics(topics):
    bs = [t if isinstance(t, bytes) else t.encode() for t in topics]
    offs = np.zeros(len(bs) + 1, dtype=np.uint32)
    offs[1:] = np.cumsum([len(b) for b in bs], dtype=np.uint64)
    return np.frombuffer(b"".join(bs), dtype=np.uint8).copy() if bs else np.zeros(0, np.uint8), offs


def _b(s) -> bytes:
    return s.encode() if isinstance(s, str) else s


def sized_topics(n: int, total: int, tag: str) -> list[bytes]:
    """n valid topics under the root `stage` with exactly `total` text bytes.  Every topic has levels of 26..29 bytes (the
    inline / pool boundary of the dictionary) and one level longer than 28 bytes (finished byte by byte by the tokeniser)."""
    base = total // n
    assert base >= 48, "topics of at least 48 bytes"
    out = []
    for i in range(n):
        ln = base + (1 if i < total - base * n else 0)
        head = f"stage/{tag}{i % 4}/" + "k" * (26 + i % 4) + "/"
        tail = ln - len(head)
        out.append((head + ("q%d" % i).ljust(tail, "z")).encode())
    assert sum(len(t) for t in out) == total
    return out


def subscription_corpus(shallow: bool = False) -> Corpus:
    """The boundary corpus.  shallow=True: the trie of a second engine (wide / Bloom-colliding nodes, 8-slot windows),
    whose max_depth is 3, so 12-level topics stay on the fast path there."""
    c = Corpus()
    add = c.adds.append
    for f, v in ROOT_WILD:
        add((f, v))
    groups: dict[str, list[Case]] = {}

    # ---- trie structure: a node with more than WIDE_FANOUT children (child filter), one with 30 (saturated Bloom mask),
    #      probed for dictionary tokens that are no child of theirs
    g = groups["structure"] = []
    for i in range(60):
        add((f"wide/c{i}", 100 + i))
    for i in range(30):
        add((f"bloom/c{i}", 200 + i))
    for i in range(40):
        add((f"dictm/m{i}", 300 + i))
    add(("wide/c7/#", 400))
    g += [Case(_b(f"wide/c{i}"), W + 1 + (i == 7)) for i in range(60)] + [Case(_b(f"wide/m{i}"), W) for i in range(40)]   # (wide/c7/# matches its parent)
    g += [Case(_b(f"bloom/c{i}"), W + 1) for i in range(30)] + [Case(_b(f"bloom/m{i}"), W) for i in range(40)]
    g += [Case(_b(f"dictm/m{i}"), W + 1) for i in range(0, 40, 5)]
    g += [Case(_b("wide/c7/" + "/".join("abcdefghij")), W + 1)]                      # 12 levels: wide/c7/#
    if shallow:
        c.max_depth = 3
        c.batches["main"] = groups["structure"]
        return c

    # ---- matched value sets per topic: 8 / 9 (first spill row), 32 (last spill row), 33 (deferred)
    g = groups["sets"] = []
    for k in (K2_SMEM_DESCS, K2_SMEM_DESCS + 1, K2_SMEM_DESCS + K2_POOL_ROWS, K2_SMEM_DESCS + K2_POOL_ROWS + 1):
        lit = ["a", "b", "c", "d", "e"]
        hashes = [f"ms{k}/" + "".join(x + "/" for x in lit[:j]) + "#" for j in range(6)]
        combos = [f"ms{k}/" + "/".join("+" if m >> i & 1 else lit[i] for i in range(5)) for m in range(32)]
        own = (hashes + combos)[:k - W]
        for i, f in enumerate(own):
            add((f, 10000 * k + i))
            if i % 3 == 0:
                add((f, 10000 * k + i + 5000))                                     # some sets of two values
        g.append(Case(_b(f"ms{k}/a/b/c/d/e"), k))                                 # every filter of the case matches it

    # ---- value-set sizes: single values 0 and 2^32-1, two values; 65534 members (largest in-line set) and 65535 (CNT_BIG)
    g = groups["values"] = []
    add(("vs/zero", 0)); add(("vs/max", 0xFFFFFFFF)); add(("vs/two", 1)); add(("vs/two", 2))
    g += [Case(b"vs/zero", W + 1), Case(b"vs/max", W + 1), Case(b"vs/two", W + 1), Case(b"vs/none", W)]
    c.bulk.append(("big/+", 1_000_000, CNT_BIG - 1))
    c.bulk.append(("huge/+", 2_000_000, CNT_BIG))

    # ---- levels: 7 / 8 on the fast path, 9 and deeper deferred, deeper than the trie's max_depth (14)
    g = groups["levels"] = []
    lv = [str(i) for i in range(1, 40)]
    add(("lv/#", 500))
    for d in (7, 8, 9):
        add(("lv/" + "/".join(lv[:d - 1]), 500 + d))
    add(("lv/" + "/".join(["+"] * 8), 510))
    add(("deep/" + "/".join(["+"] * 12) + "/#", 520))                              # 14 levels: the trie's max_depth
    c.max_depth = 14
    g += [Case(_b("lv/" + "/".join(lv[:6])), W + 2), Case(_b("lv/" + "/".join(lv[:7])), W + 2), Case(_b("lv/" + "/".join(lv[:8])), W + 3)]
    g += [Case(_b("lv/" + "/".join(lv[:39])), W + 1), Case(_b("deep/" + "/".join(lv[:19])), W + 1), Case(_b("deep/" + "/".join(lv[:12])), W + 1)]
    g += [Case(_b("deep/" + "/".join(lv[:11])), W)]                               # 12 levels: one short of the filter

    # ---- level strings: 26 / 27 (last in-line) / 28 / 29 / long, near misses of the same length, multi-byte UTF-8, blank
    #      levels, `$` roots, literal '+' / '#' levels, wildcard characters inside a level (invalid)
    g = groups["strings"] = []
    for n in (26, 27, 28, 29, 40, 100):
        s = "".join(chr(97 + (i * 7 + n) % 26) for i in range(n))
        add((f"str/{s}", 600 + n))
        add((f"str/{s}/t", 700 + n))
        miss = s[:-1] + ("A" if s[-1] != "A" else "B")
        g += [Case(_b(f"str/{s}"), W + 1), Case(_b(f"str/{s}/t"), W + 1), Case(_b(f"str/{miss}"), W), Case(_b(f"str/{s[:-1]}"), W)]
    add(("utf/é/😀/ü", 800)); add(("blank//x", 801)); add(("blank/+/x", 802)); add(("blank/#", 803))
    add(("$SYS/#", 804)); add(("$SYS/+", 805)); add(("$SYS/a", 806)); add(("lit/+", 807)); add(("lit/#", 808))
    g += [Case("utf/é/😀/ü".encode(), W + 1), Case("utf/é/😀/u".encode(), W), Case(b"blank//x", W + 3), Case(b"blank//", W + 1),
          Case(b"", W), Case(b"/", W), Case(b"$SYS/a", 3), Case(b"$SYS", 1), Case(b"$x/a", 0), Case(b"$SYS/a/$b", None),
          # a literal '+' / '#' level also looks up the wildcard child of that name: lit/+ twice; lit/# and +/# twice each
          Case(b"lit/+", W + 3), Case(b"lit/#", W + 4),Case(b"lit/a+b", None), Case(b"lit/#/x", None), Case(b"lit/b#", None)]

    # ---- extra trees (gm_match_batch_trees); tree 9 does not exist
    c.trees = {1: [("#", 11), ("ms8/#", 12), ("+/a/#", 13)], 5: [("$SYS/#", 51), ("wide/+", 52), ("lit/+", 53)]}

    main = [x for name in ("structure", "sets", "values", "levels", "strings") for x in groups[name]]
    c.batches["main"] = main
    c.batches["big_tile"] = [Case(_b(f"big/t{i}"), W + 1) for i in range(32)]            # one full tile over the 65534-member set
    c.batches["huge"] = [Case(b"huge/x", W + 1, big=True), Case(b"big/x", W + 1), Case(b"huge", W), Case(b"vs/two", W + 1)]
    for n in (1, 31, 32, 33, 64, 65, 511, 512, 513, 2048, 2049):                          # batch shapes: tiles, CTAs, small-graph tiers
        c.batches[f"n{n}"] = [main[(i * 7) % len(main)] for i in range(n)]
    # tokeniser stage: CTA 0's 16-byte aligned slice is exactly TOK_STAGE_BYTES (staged), CTA 1's 16 bytes more (global loads)
    c.batches["stage"] = [Case(t, W + 1) for t in sized_topics(TOK_THREADS, TOK_STAGE_BYTES, "s") + sized_topics(TOK_THREADS, TOK_STAGE_BYTES + 16, "t")]
    _, so = c.packed("stage")
    assert so[TOK_THREADS] == TOK_STAGE_BYTES and so[2 * TOK_THREADS] - so[TOK_THREADS] == TOK_STAGE_BYTES + 16
    # small-graph text edges: exactly the tier's text capacity, and one byte more
    for (cap_n, cap_blob, _), tier in zip(SMALL_TIERS, (0, 1)):
        c.batches[f"text{tier}_at"] = [Case(t, W + 1) for t in sized_topics(cap_n, cap_blob, "a")]
        c.batches[f"text{tier}_over"] = [Case(t, W + 1) for t in sized_topics(cap_n, cap_blob + 1, "b")]
        assert c.packed(f"text{tier}_at")[1][-1] == cap_blob and c.packed(f"text{tier}_over")[1][-1] == cap_blob + 1
    # small-graph output edges: exactly the tier's output capacity in ids, and one id more (-> the pipelined path)
    add(("stage/#", 900))
    for f, k in (("outs/v62", 62), ("outs/v63", 63)):
        for v in range(k):
            add((f, 20000 + 100 * k + v))
    for (cap_n, _, cap_out), tier in zip(SMALL_TIERS, (0, 1)):
        assert cap_n * (W + 62) == cap_out                                       # outs/v62 yields W + 62 ids, outs/v63 one more
        c.batches[f"out{tier}_at"] = [Case(b"outs/v62", W + 1)] * cap_n
        c.batches[f"out{tier}_over"] = [Case(b"outs/v62", W + 1)] * (cap_n - 1) + [Case(b"outs/v63", W + 1)]
    return c


def check_against_oracle(c: Corpus, tree: orc.TopicTree | None = None):
    """Every distinct topic of every batch, one at a time: F and validity as the case states."""
    tree = tree or c.load_oracle()
    seen = {}
    for name, cases in c.batches.items():
        for x in cases:
            if x.topic in seen:
                assert seen[x.topic] == x.F, (name, x.topic)
                continue
            seen[x.topic] = x.F
            want = tree.match_batch(*pack_topics([x.topic]), want_ids=False)
            if x.F is None:
                assert want["counts"][0] < 0, x.topic
            else:
                assert want["counts"][0] >= 0 and want["counters"]["F"] == x.F, (x.topic, want["counters"]["F"], x.F)


def retained_corpus(seed: int = 8):
    """Retained topics and filters of up to 14 levels (levels >= 8 live in the level-major token array), literal '+' / '#'
    levels that shadow wildcard expansion, `$` roots, removals.  -> (ops [(op, topic, value)], filters)"""
    rng = random.Random(seed)

    def deep_topic():
        lv = [rng.choice(["a", "b", "c", "", "dd"]) if rng.random() < 0.93 else rng.choice(["+", "#"]) for _ in range(rng.randint(1, 14))]
        if rng.random() < 0.1:
            lv[0] = "$x"
        return "/".join(lv)

    def deep_filter():
        lv = [rng.choice(["a", "b", "c", "", "dd", "+", "+"]) for _ in range(rng.randint(1, 14))]
        if rng.random() < 0.3:
            lv[-1] = "#"
        if rng.random() < 0.05:
            lv[0] = "$x"
        return "/".join(lv)

    ops = []
    for i in range(5000):
        ops.append(("set", deep_topic(), i))
        if i % 7 == 3:
            ops.append(("remove", deep_topic(), 0))
    ops += [("set", t, 90000 + i) for i, t in enumerate(["a/+", "a/#", "+", "#", "$SYS/x", "$SYS/+", "a/+/b", "a/b/" + "/".join(["c"] * 11)])]
    filters = [deep_filter() for _ in range(1200)] + ["#", "+/#", "+/+/+/+/+/+/+/+/+/#", "a/a/a/a/a/a/a/a/a/a/+", "/".join(["+"] * 12),
                                                      "a/+", "a/#", "+", "$SYS/#", "$SYS/+", "+/+", "a/b/" + "/".join(["c"] * 11), "a/b/+/#"]
    return ops, filters


def load_retained(ops, eng_set, eng_remove):
    """Apply the ops to an engine (callables returning True when accepted) and to the oracle; -> oracle RetainTree."""
    rt = orc.RetainTree()
    for op, t, v in ops:
        if op == "set":
            if eng_set(t, v):
                rt.insert(t, v)
        elif eng_remove(t):
            rt.remove(t)
    return rt
