"""Cases of the message store (gm_msgstore_*), run against tests/_msgstore_oracle.py on the CPU emulation
(test_msgstore_cpu.py) and through the real ABI on the GPU (test_gpu_msgstore.py).

A store adapter S offers store(topic, handle, expiry, forwarded), get(now, filters, clients, groups, cap=None) ->
(rc, needed, lists) with lists[i] sorted or None for an invalid filter, remove_expired(now, cap) -> handles, stats() -> dict.
Clients are strings; forwarded is [(client, None | (filter, group))]; groups[i] is None or query i's shared group."""
from __future__ import annotations

import random


NOW = 1_760_000_000_000
LATER = NOW + 3_600_000


def check(S, ref, now, queries, cap=None):
    """one batch through both; queries = [(filter, client, group)]; returns the lists"""
    fs, cs, gs = [q[0] for q in queries], [q[1] for q in queries], [q[2] for q in queries]
    rc, needed, got = S.get(now, fs, cs, gs, cap)
    assert rc == 0, (rc, needed)
    want = ref.get_batch(now, fs, cs, gs)
    assert got == want, [(i, q, g, w) for i, (q, g, w) in enumerate(zip(queries, got, want)) if g != w][:5]
    return got


def put(S, ref, topic, h, expiry=LATER, fwd=()):
    S.store(topic, h, expiry, list(fwd))
    ref.set(topic, h, expiry, list(fwd))


def case_new_and_repeated(S, ref):
    put(S, ref, "a/b", 1)
    put(S, ref, "a/c", 2)
    assert check(S, ref, NOW, [("a/+", "A", None)]) == [[1, 2]]
    assert check(S, ref, NOW, [("a/+", "A", None), ("a/b", "B", None)]) == [[], [1]]
    assert check(S, ref, NOW, [("a/#", "A", None)]) == [[]]


def case_store_time_marks(S, ref):
    put(S, ref, "s/x", 10, fwd=[("A", None), ("B", ("s/+", "g"))])
    got = check(S, ref, NOW, [("s/x", "A", None), ("s/+", "C", "g"), ("s/x", "B", None), ("s/x", "D", None)])
    assert got == [[], [], [], [10]]


def case_group_under_another_filter(S, ref):
    put(S, ref, "g/1", 20)
    got = check(S, ref, NOW, [("g/+", "A", "grp"), ("g/#", "B", "grp"), ("g/+", "C", "grp")])
    assert got == [[20], [20], []]


def case_shared_then_plain_same_client(S, ref):
    put(S, ref, "p/1", 30)
    assert check(S, ref, NOW, [("p/+", "A", "g"), ("p/1", "A", None), ("p/+", "B", None)]) == [[30], [], [30]]


def case_expiry_edges(S, ref):
    put(S, ref, "e/now", 40, expiry=NOW)
    put(S, ref, "e/past", 41, expiry=NOW - 1)
    put(S, ref, "e/late", 42, expiry=NOW + 1)
    assert check(S, ref, NOW, [("e/+", "A", None)]) == [[40, 42]]
    assert check(S, ref, NOW, [("e/+", "B", None)]) == [[40, 42]]
    assert check(S, ref, NOW + 1, [("e/+", "C", None)]) == [[42]]
    assert sorted(S.remove_expired(NOW, 10)) == sorted(ref.remove_expired(NOW)) == [40, 41]      # expiry_time_at <= now


def case_append_rule(S, ref):
    for h, t in ((50, "a/b"), (51, "a"), (52, "$SYS/x"), (53, "a/b/c"), (5, "a"), (54, ""), (55, "a/"), (56, "/x")):
        put(S, ref, t, h)
    fs = ["a/b", "a/#", "#", "+", "$SYS/#", "a/5/#", "", "a/", "+/+", "/#", "a/b/#", "$SYS/+"]
    for i, f in enumerate(fs):
        check(S, ref, NOW, [(f, f"c{i}", None)])
    got = check(S, ref, NOW, [("a/5/#", "fresh", None)])
    assert got == [[5]]                 # message 5 published to `a` is kept under a/5


def case_invalid_row(S, ref):
    put(S, ref, "i/1", 60)
    rc, needed, got = S.get(NOW, ["i/+", "i/#/x", "i/+x"], ["A", "B", "C"], [None, None, None])
    assert rc == 0 and got == [[60], None, None]
    ref.get_batch(NOW, ["i/+"], ["A"], [None])
    assert check(S, ref, NOW, [("i/+", "B", None), ("i/+", "C", None)]) == [[60], [60]]


def case_chain(S, ref):
    put(S, ref, "c/1", 70)
    # a share key names (filter, group): q1 / q2 share (c/+, S1), q2 / q3 client B, q3 / q4 (c/#, S2), q4 / q5 client C
    q = [("c/+", "A", "S1"), ("c/+", "B", "S1"), ("c/#", "B", "S2"), ("c/#", "C", "S2"), ("c/1", "C", None)]
    assert check(S, ref, NOW, q) == [[70], [], [70], [], [70]]


def case_big_group(S, ref, members=1000):
    for h in range(80, 90):
        put(S, ref, f"big/{h}", h)
    q = [("big/+", f"m{i}", "grp") for i in range(members)]
    got = check(S, ref, NOW, q)
    assert got[0] == list(range(80, 90)) and all(g == [] for g in got[1:])


def case_capacity(S, ref):
    for h in range(100, 110):
        put(S, ref, f"cap/{h}", h)
    q = [("cap/+", "A", None), ("cap/#", "B", "g"), ("cap/+", "A", None)]
    rc, needed, _ = S.get(NOW, [x[0] for x in q], [x[1] for x in q], [x[2] for x in q], cap=0)
    assert rc != 0 and needed == 20
    rc, needed2, _ = S.get(NOW, [x[0] for x in q], [x[1] for x in q], [x[2] for x in q], cap=needed - 1)
    assert rc != 0 and needed2 == needed
    assert check(S, ref, NOW, q, cap=needed) == [list(range(100, 110)), list(range(100, 110)), []]
    assert check(S, ref, NOW, q) == [[], [], []]


def case_restore_after_sweep(S, ref):
    put(S, ref, "r/1", 120, expiry=NOW - 10, fwd=[("A", None)])
    put(S, ref, "r/2", 121, expiry=NOW + 10)
    assert check(S, ref, NOW - 20, [("r/+", "B", "g")]) == [[120, 121]]
    assert sorted(S.remove_expired(NOW, 100)) == sorted(ref.remove_expired(NOW)) == [120]
    assert S.stats()["retired"] == 1
    put(S, ref, "r/1", 120, expiry=LATER)          # the same handle again: no marks
    assert check(S, ref, NOW, [("r/+", "A", None), ("r/+", "C", "g")]) == [[120, 121], [120]]
    st = S.stats()
    assert st["retired"] == 0 and st["purges"] >= 1


def case_growth(S, ref, steps=12, per_step=50):
    clients = [f"cl{i}" for i in range(steps)]
    h = 1000
    for i, c in enumerate(clients):
        for _ in range(per_step):
            put(S, ref, f"gr/{h % 7}", h, fwd=[(f"k{h % 5}", None)])
            h += 1
        check(S, ref, NOW, [("gr/#", c, "G" if i % 3 == 0 else None)])
    st = S.stats()
    assert st["rehashes"] >= 3 and st["mark_slots"] >= 2 * st["marks"]
    q = [("gr/#", c, None) for c in clients] + [("gr/#", f"k{k}", None) for k in range(5)]
    check(S, ref, NOW, q)
    # every mark survived the rebuilds: nobody gets anything again
    assert check(S, ref, NOW, q) == [[]] * len(q)


ALL = [case_new_and_repeated, case_store_time_marks, case_group_under_another_filter, case_shared_then_plain_same_client, case_expiry_edges,
       case_append_rule, case_invalid_row, case_chain, case_big_group, case_capacity, case_restore_after_sweep, case_growth]


def random_rounds(S, ref, orc_seed: int, rounds: int, per_round: int, batch: int, n_clients: int, n_groups: int, handle_base: int = 1):
    """seeded differential: stores with marks, batched gets with repeated clients and groups, sweeps with an advancing now"""
    rng = random.Random(orc_seed)
    now = NOW
    h = handle_base
    levels = [["r0", "r1", "r2"], ["s0", "s1", "s2", "s3"], ["d0", "d1", "d2", "d3", "d4"]]
    for _ in range(rounds):
        for _ in range(per_round):
            t = "/".join(rng.choice(lv) for lv in levels[:rng.randrange(1, 4)])
            fwd = [(f"c{rng.randrange(n_clients)}", None if rng.random() < 0.6 else (rng.choice(["r0/#", "+/s1/#", "#"]), f"g{rng.randrange(n_groups)}"))
                   for _ in range(rng.randrange(3))]
            put(S, ref, t, h, expiry=now + rng.randrange(-100, 2000), fwd=fwd)
            h += 1
        q = []
        for _ in range(batch):
            f = rng.choice(["#", "r0/#", "+/s1/#", "r1/+", "r2/s3", "+/+/d1", "r0/s0/+", "+"])
            g = None if rng.random() < 0.5 else f"g{rng.randrange(n_groups)}"
            q.append((f, f"c{rng.randrange(n_clients)}", g))
        check(S, ref, now, q)
        now += rng.randrange(0, 300)
        got = S.remove_expired(now, 1 << 20)
        assert sorted(got) == sorted(ref.remove_expired(now))
    return h
