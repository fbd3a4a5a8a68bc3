"""Boundary corpus of the retained-message lookup (k_retain_init, k_retain_round, k_retain_scan, k_retain_expand).

Deterministic, like `_edges.subscription_corpus()`: every case reaches its edge by construction and states what it expects.
Results come from the oracle's RetainTree; what the corpus adds is, for every single-filter shape case, the number of tasks
each round must queue (`RQuery.tasks`: entry 0 = what k_retain_init queued, entry l + 1 = what round l queued — the numbering
of the engine's `retain stats` line; rounds beyond the tuple must queue nothing).  The counts are derived by hand in the
comments below from the rules of retain_kernels.cuh, not computed by a model of the kernel.

Two trees:
  * `retained_edge_corpus()` has no literal `#` level anywhere, so the root keeps its `#` range shortcut (root_plain_val_hi);
  * `retained_lit_hash_corpus()` holds a chain with a literal `#` level at the bottom, which sends `#` down the walk (mode 2).

The constants mirror rmqtt_b200/csrc/retain_kernels.cuh and retain_tree.h; `check_constants` asserts the cases depend on them.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

RTASK_CHUNK = 256        # child-block entries per task (retain_kernels.cuh)
RINLINE_KIDS = 8         # a '+' / shadowed '#' over at most this many children is expanded in place ...
RINLINE_DEPTH = 4        # ... in at most this many nested frames (retain_chain)
RLIST = 256              # stage-B survivor list of k_retain_round (one entry per child of a task)
RQ = 64                  # queue slices; the scratch is split into RQ slices of cap / RQ entries
SCAN_THREADS = 1024      # k_retain_scan: one CTA, ceil(nq / 1024) filters per thread
INIT_THREADS = 256       # k_retain_init: one thread per filter, 256 per CTA
VMAX = 0xFFFFFFFF

# Child-block sizes of the shape nodes w/k<k> and the tasks `w/k<k>/+` queues in k_retain_init: at most RINLINE_KIDS
# children are expanded in place (0 tasks); above, one task per RTASK_CHUNK children, the last one short.
#   8 -> in place; 9 -> 1 task of 9; 255, 256 -> 1; 257 -> 256 + 1; 512 -> 2 x 256; 513 -> 2 x 256 + 1;
#   65537 -> 256 x 256 + 1 = 257 tasks
SHAPE_TASKS = {8: 0, 9: 1, 255: 1, 256: 1, 257: 2, 512: 2, 513: 3, 65537: 257}
BIG = 65537
SURVIVORS = (0, 1, 255, 256)          # children of s/n<m> (256 in all) under which the literal `lit` exists
N_BLOOM_Q = 32                        # query literals q0..q31 probed below bl/mid (some bit-clear, some false positives)
BATCH_SHAPES = (1, 255, 256, 257, 1023, 1024, 1025, 2048, 2049, 4097)
INVALID = ("a/#/b", "a+", "#/x")      # Topic::from_str fails: status and count come from the oracle


@dataclass
class RQuery:
    filt: str
    tasks: tuple | None = None        # tasks queued per round (see module doc); None = not stated
    heavy: bool = False               # expands the 65537-child node or the whole tree: not drawn into the batch shapes


@dataclass
class RCorpus:
    sets: list = field(default_factory=list)       # (topic, value), in this order
    bulk: list = field(default_factory=list)       # (topic, value) of the 65537-child node, loaded with retain_bulk_load
    queries: list = field(default_factory=list)    # [RQuery]

    def all_topics(self):
        return self.sets + self.bulk

    def filters(self, heavy=True):
        return [q.filt for q in self.queries if heavy or not q.heavy]

    def stated(self):
        return [q for q in self.queries if q.tasks is not None]

    def batch(self, n: int) -> list[str]:
        """A batch of n filters drawn from the light cases, with an invalid filter or the empty filter every 97th row
        (a batch of one is a single shape case)."""
        light = self.filters(heavy=False)
        bad = list(INVALID) + [""]
        return [bad[(i // 97) % len(bad)] if i % 97 == 5 else light[(i * 7) % len(light)] for i in range(n)]

    def load_oracle(self, orc):
        rt = orc.RetainTree()
        for t, v in self.all_topics():
            rt.insert(t, v)
        return rt

    def value_of(self, topic: str) -> int:
        for t, v in self.all_topics():
            if t == topic:
                return v
        raise KeyError(topic)


def pack(strings):
    bs = [s.encode() if isinstance(s, str) else s for s in strings]
    offs = np.zeros(len(bs) + 1, dtype=np.uint32)
    if bs:
        offs[1:] = np.cumsum([len(b) for b in bs], dtype=np.uint64)
    return (np.frombuffer(b"".join(bs), dtype=np.uint8).copy() if bs else np.zeros(0, np.uint8)), offs


def retained_edge_corpus() -> RCorpus:
    c = RCorpus()
    nv = [1000]

    def put(t, v=None):
        if v is None:
            nv[0] += 1
            v = nv[0]
        c.sets.append((t, v))

    Q = c.queries.append
    # ---- roots whose tokens interleave: dictionary tokens are handed out in order of first appearance, so `$a` lies between
    #      r1 and r2 in token order while the device block keeps plain children first
    for t in ("r1/x", "$a/x", "r2/x", "$b/x", "r3/x", "$a", "$b", "$a/y/z"):
        put(t)
    put("vz", 0)
    put("vm", VMAX)
    # ---- child-block sizes: w/k<k> with k valued leaf children.  Own values: w/k9 = 2^32-1, w/k257 = 0 (X/# skips them by
    #      val_lo + 1 and emits them as the parent match), w/k8 none
    for k in SHAPE_TASKS:
        if k == 9:
            put("w/k9", VMAX)
        elif k == 257:
            put("w/k257", 0)
        elif k != 8:
            put(f"w/k{k}")
        if k == BIG:
            c.bulk += [(f"w/k{k}/c{i}", 2_000_000 + i) for i in range(k)]
        else:
            for i in range(k):
                put(f"w/k{k}/c{i}")
        T = SHAPE_TASKS[k]
        # `+` / `+/zz`: k_retain_init reaches w/k<k> by exact steps and queues T tasks there; round 0 ends every child (the
        # filter ends, or the child is a leaf and `zz` cannot follow) and queues nothing.  `#`: no literal `#` below, one range
        Q(RQuery(f"w/k{k}/+", (T,), heavy=k == BIG))
        Q(RQuery(f"w/k{k}/+/zz", (T,), heavy=k == BIG))
        Q(RQuery(f"w/k{k}/#", (0,), heavy=k == BIG))
    put("zz/top")                                   # (interns `zz`: a literal the dictionary knows)
    # ---- stage-B survivor lists: s/n<m> has 256 valued children c<i>; the first m of them have a valued child `lit`, which
    #      has a valued child `z`.  One task of 256 children (k_retain_init); stage A puts the m children whose Bloom mask
    #      admits `lit` on the list (0, 1, 255 or all RLIST = 256); stage B probes them; nothing is queued below.
    for m in SURVIVORS:
        for i in range(256):
            put(f"s/n{m}/c{i}")
            if i < m:
                put(f"s/n{m}/c{i}/lit")
                put(f"s/n{m}/c{i}/lit/z")
        Q(RQuery(f"s/n{m}/+/lit", (1, 0)))            # the filter ends at a stage-B child
        Q(RQuery(f"s/n{m}/+/lit/z", (1, 0)))          # two exact levels: the list is probed twice
        Q(RQuery(f"s/n{m}/+/lit/#", (1, 0)))          # stage-B parent `#` (lit's own value), then lit's range
        Q(RQuery(f"s/n{m}/+/#", (1, 0)))              # stage-A parent `#`, then every child's range
    # ---- nesting: n/<a|b>^6, every node below n valued.  `+` over 2 children is expanded in place; the four frames are
    #      n's block (level 1), level 2, 3 and 4 blocks ... so at each of the 16 level-4 nodes all RINLINE_DEPTH frames are
    #      in use when the 5th `+` comes: 16 tasks from k_retain_init.  Round 0 ends at level 5 (filter of 6 levels), or
    #      expands level 6 in place from a fresh stack (7 and 8 levels): nothing more is queued.
    front = ["n"]
    for _ in range(6):
        front = [f"{p}/{x}" for p in front for x in ("a", "b")]
        for t in front:
            put(t)
    Q(RQuery("n/+/+/+/+", (0,)))                      # 4 frames exactly: no task
    Q(RQuery("n/+/+/+/+/+", (16, 0)))
    Q(RQuery("n/+/+/+/+/+/+", (16, 0)))
    Q(RQuery("n/+/+/+/+/+/+/+", (16, 0)))             # level-6 leaves cannot continue
    Q(RQuery("n/+/+/+/+/+/#", (16, 0)))               # stage-A parent `#` over level 5, ranges below
    Q(RQuery("n/a/+/+/+/+", (0,)))                    # one exact step first: 4 frames, level 5 ends the filter
    Q(RQuery("n/+/b/+/a/+/+", (0,)))                  # exact levels between the `+`: frames at levels 1, 3, 5 only
    # ---- parent `#` and filter end at each site: exact step (pa), in-place loop (pi, 3 children), stage A (pA, 20 children);
    #      stage B is s/n<m>/+/lit/# and s/n<m>/+/lit above
    put("pa/v"); put("pa/v/x")
    for i in range(3):
        put(f"pi/c{i}"); put(f"pi/c{i}/k")
    for i in range(20):
        put(f"pA/c{i}"); put(f"pA/c{i}/k")
    Q(RQuery("pa/v/#", (0,))); Q(RQuery("pa/v", (0,))); Q(RQuery("pa/v/x", (0,)))
    Q(RQuery("pi/+/#", (0,))); Q(RQuery("pi/+", (0,))); Q(RQuery("pi/+/k", (0,)))
    Q(RQuery("pA/+/#", (1, 0))); Q(RQuery("pA/+", (1, 0))); Q(RQuery("pA/+/k", (1, 0)))
    # ---- Bloom masks below bl (3 children, expanded in place, so the in-place loop reads each child's mask from the child
    #      block): bl/sat has 256 children (mask saturated), bl/mid 12, bl/one 1.  The literals q<j> exist in the dictionary
    #      (bq/q<j>); `bloom_proof` finds among them a bit-clear one and a false positive of bl/mid from the image.
    put("bl/sat"); put("bl/mid")
    for i in range(256):
        put(f"bl/sat/c{i}")
    for i in range(12):
        put(f"bl/mid/m{i}")
    put("bl/one/m0")
    for j in range(N_BLOOM_Q):
        put(f"bq/q{j}")
        Q(RQuery(f"bl/+/q{j}", (0,)))
    Q(RQuery("bl/+/m3", (0,))); Q(RQuery("bl/+/m0", (0,))); Q(RQuery("bl/sat/c200", (0,)))
    # ---- block that in-place edits grow (1 child now)
    put("gr/x0")
    # ---- roots
    for f in ("#", "+/#", "+/+/#"):
        Q(RQuery(f, heavy=True))
    for f in ("+", "+/x", "$a/#", "$a/+", "$b/x", "$a", "$", "vz", "vm", "vz/#", "vm/#", "w/k9", "w/k257"):
        Q(RQuery(f))
    for f in INVALID + ("",):
        Q(RQuery(f))
    return c


def retained_lit_hash_corpus() -> RCorpus:
    """h/<a|b>^6/# with a literal `#` level under every level-6 node: every node of the chain (and the root) has
    RF_SUB_LIT_HASH, so `h/#` walks in mode 2."""
    c = RCorpus()
    nv = [5000]

    def put(t, v=None):
        if v is None:
            nv[0] += 1
            v = nv[0]
        c.sets.append((t, v))

    for t in ("r1/x", "$a/x", "r2/x", "$a", "vz", "h"):
        put(t)
    front = ["h"]
    for _ in range(6):
        front = [f"{p}/{x}" for p in front for x in ("a", "b")]
        for t in front:
            put(t)
    for t in front:
        put(f"{t}/#")
    # h/#: h by an exact step (its own value as the parent match), then mode 2 in place through levels 1..4 (the four
    # frames); each of the 16 level-4 nodes queues its 2 children: 16 tasks.  Round 0 takes level 5 into a fresh stack,
    # level 6 in place, and the literal `#` child by an exact step: nothing more is queued.
    # h/a/# and h/+/#: the frames start one level lower (levels 2..5 below h), so the 16 nodes of level 5 below h/a — and
    # the 16 of level 4 below h for h/+/# — spill.  h/+/+/+/+/+/+/#: the 16 level-4 nodes spill the 5th `+`.
    c.queries += [RQuery("h/#", (16, 0)), RQuery("h/a/#", (16, 0)), RQuery("h/+/#", (16, 0)), RQuery("h/a/a/a/a/a/a/#", (0,)),
                  RQuery("h/+/+/+/+/+/+/#", (16, 0))]
    c.queries += [RQuery(f) for f in ("#", "+", "+/#", "$a/#", "h/a/b/a/b/a/#", "r1/#")]
    c.queries += [RQuery(f) for f in INVALID + ("",)]
    return c


def check_constants():
    """The cases sit on the boundaries the constants define."""
    assert SHAPE_TASKS[RINLINE_KIDS] == 0 and SHAPE_TASKS[RINLINE_KIDS + 1] == 1
    assert SHAPE_TASKS[RTASK_CHUNK] == 1 and SHAPE_TASKS[RTASK_CHUNK + 1] == 2 and SHAPE_TASKS[2 * RTASK_CHUNK + 1] == 3
    assert SHAPE_TASKS[BIG] == RTASK_CHUNK + 1 and BIG == RTASK_CHUNK * RTASK_CHUNK + 1
    assert max(SURVIVORS) == RLIST == RTASK_CHUNK
    assert 2 ** RINLINE_DEPTH == 16               # level-4 nodes of the 2-ary chains: each spills one task
    for n in (INIT_THREADS - 1, INIT_THREADS, INIT_THREADS + 1, SCAN_THREADS, SCAN_THREADS + 1, 2 * SCAN_THREADS + 1):
        assert n in BATCH_SHAPES


# ---- reading the retained image (Engine.debug_tables(): rnodes / rkids, 8 words each) ----------------------------------
RNK_MASK = 0x0FFFFFFF


def retain_mask_bit(token: int) -> int:
    """retain_tree.h retain_mask_bit: one of 32 bits for a child token."""
    return 1 << (((token * 0x9E3779B1) & 0xFFFFFFFF) >> 27)


class Image:
    """Child blocks of the exported image, found by the children's values (every corpus node has its own value)."""

    def __init__(self, rnodes: np.ndarray, rkids: np.ndarray):
        self.rnodes, self.rkids = rnodes, rkids

    def block(self, dev: int) -> np.ndarray:
        fk, nk = int(self.rnodes[dev][0]), int(self.rnodes[dev][1])
        return self.rkids[fk:fk + nk]

    def entry_by_value(self, value: int) -> np.ndarray:
        """The child-block entry {token, child, first_kid, nk_flags, val, val_lo, val_hi, mask} of the valued node."""
        live = self.rkids[(self.rkids[:, 4] == value) & ((self.rkids[:, 3] >> 31) & 1 == 1)]
        assert len(live) >= 1, value
        return live[0]

    def token_of_value(self, value: int) -> int:
        return int(self.entry_by_value(value)[0])


def bloom_proof(c: RCorpus, img: Image) -> dict:
    """Proves from the image that the Bloom cases exist: bl/sat's mask is saturated; among q0..q31 at least one has its bit
    clear in bl/mid's mask and at least one is a false positive (bit set, no such child).  -> {"clear": [j], "fp": [j]}"""
    sat, mid = img.entry_by_value(c.value_of("bl/sat")), img.entry_by_value(c.value_of("bl/mid"))
    assert int(sat[7]) == 0xFFFFFFFF, hex(int(sat[7]))
    mid_mask = int(mid[7])
    mid_kids = {int(e[0]) for e in img.block(int(mid[1]))}
    assert len(mid_kids) == 12
    clear, fp = [], []
    for j in range(N_BLOOM_Q):
        tok = img.token_of_value(c.value_of(f"bq/q{j}"))
        assert tok not in mid_kids
        (fp if mid_mask & retain_mask_bit(tok) else clear).append(j)
    assert clear and fp, (clear, fp)
    return {"clear": clear, "fp": fp}


def root_interleave_proof(c: RCorpus, img: Image):
    """The root block holds plain children first although a `$` root's token lies between two plain ones."""
    root = [int(e[0]) for e in img.block(0)]
    dollar = [img.token_of_value(c.value_of(t)) for t in ("$a", "$b")]
    k = len(root) - len(dollar)
    assert sorted(root[k:]) == sorted(dollar), (root, dollar)           # `$` children last ...
    assert min(root[:k]) < min(dollar) < max(root[:k]), (root, dollar)  # ... though their tokens are not


# ---- loading (c): in-place edits of a bulk-built image ------------------------------------------------------------------
DEEP = "dp/" + "/".join(["d"] * 15)     # 16 levels: deeper than anything in the corpus


def edit_script(clear_j: int) -> list:
    """Edits of the bulk-built edge corpus, each to be checked against the oracle after it runs:
    -> [(label, op, arg, how)]: op "set" (arg = (topic, value)), "remove" (topic), "remove_batch" ([topics]) or "compact";
    how = "patch" (edited in place: flattens unchanged, patches grow), "flatten" (the next lookup re-flattens) or None.
    `clear_j`: a query literal q<j> whose bit is clear in bl/mid's mask (bloom_proof)."""
    v = iter(range(9_000_000, 9_001_000))
    s = []
    for i in range(1, 9):                                   # gr's block: capacity 1 -> 2 -> 4 -> 8 -> 16, moved each time
        s.append((f"gr grows to {i + 1} children", "set", (f"gr/x{i}", next(v)), "patch"))
    s.append(("plain root child after the `$` roots", "set", ("pz/x", next(v)), "patch"))
    s.append(("a new `$` root", "set", ("$c/x", next(v)), "patch"))
    s.append(("a value for the valueless inner node s/n1", "set", ("s/n1", next(v)), "patch"))
    s.append(("prune pi/c0/k to a dead leaf", "remove", "pi/c0/k", "patch"))
    s.append(("revive pi/c0/k", "set", ("pi/c0/k", next(v)), "patch"))
    s.append((f"bl/mid gains q{clear_j}, whose mask bit was clear", "set", (f"bl/mid/q{clear_j}", next(v)), "patch"))
    s.append(("a topic deeper than any before", "set", (DEEP, VMAX), "patch"))
    s.append(("a literal `+` level", "set", ("lp/+/x", next(v)), "flatten"))
    s.append(("remove a batch", "remove_batch", ["vm", "w/k9", "nope/x", "pa/v/x", "a/#/b", DEEP], None))
    s.append(("compact", "compact", None, "flatten"))
    return s


REMOVE_BATCH_REMOVED = 4                 # vm, w/k9, pa/v/x and DEEP had values; nope/x did not exist, a/#/b is invalid


def edit_filters(c: RCorpus) -> list[str]:
    """The filters checked after every edit: the edited places, the root expansions, the query literals (the whole-tree `#`
    walks are checked once, after the last edit)."""
    return (["+", "+/x", "+/+", "$c/#", "$a/#", "$+", "pz/#", "gr/+", "gr/#", "gr/x8", "gr/+/y", "s/n1", "s/n1/#",
             "s/n1/+/lit", "s/+/+/lit/#", "pi/+/k", "pi/+/#", "pi/c0/#", "pi/c0/k", "dp/#", DEEP, "/".join(DEEP.split("/")[:-1]) + "/+",
             "dp/" + "/".join(["+"] * 15), "lp/+/x", "lp/#", "lp/+/+", "vm", "vm/#", "w/k9", "w/k9/#", "pa/v/#", "n/+/+/+/+/+"]
            + [f"bl/+/q{j}" for j in range(N_BLOOM_Q)] + list(INVALID) + [""])
