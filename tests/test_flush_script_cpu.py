"""CPU tier of the flush-concurrency test (tests/test_gpu_flush_concurrency.py): the writer script reaches the table
growths, value compactions, depth changes and deadlines the GPU test relies on; the expected lists derived per probe
equal a full oracle replay; and the checker rejects stale, future, torn and unflushed results."""
import os

import numpy as np
import pytest

from oracle import oracle as orc
from rmqtt_b200 import workload as wl
from rmqtt_b200.engine import Engine

import _flush_script as S
from _retain_expiry import TimedRetain


@pytest.fixture(scope="module")
def fx():
    bg = S.Background()
    ops = S.script()
    return bg, ops, S.Model(ops, bg)


def test_script_reaches_every_shipping_path_on_a_host_only_engine(fx):
    """Table growth, value compaction and max_depth are host decisions: a host-only engine takes the same ones."""
    bg, ops, model = fx
    os.environ["GM_WIN_MIN_SLOTS_LOG2"] = "3"
    try:
        eng = Engine(host_only=True)
    finally:
        os.environ.pop("GM_WIN_MIN_SLOTS_LOG2", None)
    bg.load(eng)
    start = eng.stats()
    seen = []
    prog = S.Progress()
    S.run_writer(eng, ops, prog, on_flush=lambda: seen.append((eng.stats(), eng.values_view()[2], prog.flushes_done)))
    edge = [s["edge_slots"] for s, _, _ in seen]
    dslots = [s["dict_slots"] for s, _, _ in seen]
    depth = [s["max_depth"] for s, _, _ in seen]
    epoch = [e for _, e, _ in seen]
    assert max(edge) > start["edge_slots"] and max(dslots) > start["dict_slots"]
    assert start["max_depth"] <= 8 and max(depth) > 8 and depth[-1] <= 8
    assert depth.index(max(depth)) == S.DEEP_ADD and all(d > 8 for d in depth[S.DEEP_ADD:S.COMPACT_AT])   # gm_compact lowers it
    moves = sum(1 for a, b in zip(epoch, epoch[1:]) if b != a)
    assert moves >= 3 and all(b >= a for a, b in zip(epoch, epoch[1:])), epoch      # the epoch never comes back
    assert epoch[S.COMPACT_AT] > epoch[S.COMPACT_AT - 1]                             # gm_compact rebuilt the value sets
    assert prog.mut_done == model.n and prog.flushes_done == S.K + 1        # (gm_compact flushes too)
    # the first deadline arrives while the readers of the GPU test are running, after many flushed states without one
    assert model.flushed[:model.first_deadline].sum() > S.K // 5
    st = eng.stats()
    assert st["retained_values"] == S.N_BG_RETAINED + S.W


def test_derived_expectations_equal_an_oracle_replay(fx):
    bg, ops, model = fx
    trees = {0: orc.TopicTree(), 1: orc.TopicTree()}
    trees[0].bulk_insert(*bg.subs)
    ret = TimedRetain(orc)
    for t, v in zip(wl.unpack(*bg.retained[:2]), bg.retained[2].tolist()):
        ret.set_with_timeout(t.decode(), v)
    keys = list(model.vstart)
    checked = 0

    def compare(p):
        for key in keys:
            if key[0] == "sub":
                want = trees[key[1]].matches(key[2])
            else:
                want = ret.get_message(key[2], key[1])
            assert model.expected(key, p) == tuple(want), (key, p)

    p = 0
    compare(0)
    for op in ops:
        if not S.is_mutation(op):
            continue
        k = op[0]
        if k == "add":
            trees[op[1]].insert(op[2], op[3])
        elif k == "rm":
            trees[op[1]].remove(op[2], op[3])
        elif k == "rset":
            ret.set_with_timeout(op[1], op[2], op[3])
        else:
            ret.remove(op[1])
        p += 1
        if p % 50 == 0 or p == model.n:
            compare(p)
            checked += 1
    assert checked > model.n // 50
    # every subscription probe and retained wildcard changes during the script (one that never changed could not tell two
    # states apart); a single retained topic whose message expired at NOW stays empty at NOW throughout
    assert all(len(model.vstart[k]) > 1 for k in keys if k[0] == "sub" or "+" in k[2] or "#" in k[2])


def _result(model, batch, p_of_key, bg_edit=None, invalid_status=-2):
    """A synthetic (status, counts, ids) for `batch`: probe rows from the states p_of_key(key), background rows static"""
    status, counts, ids = [], [], []
    for i, (_, _, spec) in enumerate(batch.rows):
        if spec is None:
            status.append(invalid_status); counts.append(-1)
            continue
        lst = list(model.expected(spec, p_of_key(spec))) if i in dict(batch.probes) else list(spec)
        if bg_edit is not None and i == bg_edit:
            lst[0] += 1
        status.append(0); counts.append(len(lst)); ids += lst
    return np.asarray(status, np.int32), np.asarray(counts, np.int64), np.asarray(ids, np.uint32)


def test_checker_accepts_one_state_and_rejects_torn_stale_future_and_unflushed_results(fx):
    bg, ops, model = fx
    a, b, r = ("sub", 0, "w/x"), ("sub", 0, "w/100/y"), ("ret", S.NOW, "w/#")
    j = next(i for i, l in enumerate(bg.topic_want) if l)
    batch = S.Batch([("w/x", 0, a), (bg.topics[j], 0, bg.topic_want[j]), ("w/100/y", 0, b), ("w/#/x", 0, None)])
    rbatch = S.Batch([("w/#", 0, r), ("w/a+", 0, None)])
    muts = [op for op in ops if S.is_mutation(op)]
    # p: a step boundary well inside the run; mutation p + 1 adds w/<i>/+, p + 2 adds a value of w/# (both probes change)
    p = next(q for q in range(2000, model.n) if model.flushed[q])
    assert muts[p][:2] == ("add", 0) and muts[p + 1][:3] == ("add", 0, "w/#")
    ex = lambda key, q: model.expected(key, q)
    assert ex(a, p) == ex(a, p + 1) != ex(a, p + 2) and ex(b, p) != ex(b, p + 2)

    def states(res, lo, hi, manual=False, bt=batch):
        return S.check(model, bt, *res, lo, hi, manual)

    assert p in states(_result(model, batch, lambda k: p), p - 2, p + 2).tolist()
    assert states(_result(model, batch, lambda k: p), p, p, manual=True).tolist() == [p]
    with pytest.raises(AssertionError, match="no legal state"):     # torn: w/x from p, w/100/y from p + 2
        states(_result(model, batch, lambda k: p if k == a else p + 2), p - 2, p + 4)
    with pytest.raises(AssertionError, match="no legal state"):     # stale: below lo
        states(_result(model, batch, lambda k: p), p + 2, p + 4)
    with pytest.raises(AssertionError, match="no legal state"):     # from the future: above hi
        states(_result(model, batch, lambda k: p + 4), p, p + 2)
    q = p + 2                                                       # mid-step: legal with automatic flushes only
    assert not model.flushed[q]
    assert q in states(_result(model, batch, lambda k: q), p, p + 4).tolist()
    with pytest.raises(AssertionError, match="no legal state"):
        states(_result(model, batch, lambda k: q), p, p + 4, manual=True)
    with pytest.raises(AssertionError, match="background"):         # an altered background list
        states(_result(model, batch, lambda k: p, bg_edit=1), p, p)
    with pytest.raises(AssertionError, match="invalid rows"):
        states(_result(model, batch, lambda k: p, invalid_status=0), p, p)
    # retained: the deadline rule at NOW; a handle whose deadline is between NOW and later is live at NOW, expired later
    d = next(q for q in range(model.n) if muts[q][0] == "rset" and muts[q][3] > S.NOW)
    assert muts[d][2] in ex(r, d + 1) and muts[d][2] not in ex(("ret", S.LATE, "w/#"), d + 1)
    late = (np.asarray([0, -2], np.int32), np.asarray([len(ex(("ret", S.LATE, "w/#"), d + 1)), -1]),
            np.asarray(ex(("ret", S.LATE, "w/#"), d + 1), np.uint32))
    with pytest.raises(AssertionError, match="no legal state"):
        states(late, d + 1, d + 1, bt=rbatch)
    assert states(_result(model, rbatch, lambda k: d + 1), d + 1, d + 1, bt=rbatch).tolist() == [d + 1]
