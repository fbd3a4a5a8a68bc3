"""GPU tier: single SUBSCRIBE retained lookups — the retained batcher (gm_retain_batcher_*) and the one-launch CUDA-graph path
that gm_retain_match_batch takes for batches of up to 2048 filters.  RetainStorage::get is called once per subscription in the
reference (rmqtt/src/session.rs:1336-1357); every answer must equal the oracle's RetainTree, and the graph path must give the
same spans and id multisets as the pipelined path (small_graphs 0) across flushes, compactions and scratch growth."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

import _retain_edges as R
from oracle import oracle as orc
from rmqtt_b200 import _native as N

from _gen import rand_filter, rand_topic
from test_gpu_edges import _canon, _same
from test_gpu_retain_edges import _host, _load

pytestmark = pytest.mark.gpu


def _filters(rng, c, k):
    """corpus filters plus random ones: invalid, empty, `$`-rooted, `#` and `+`-heavy"""
    fs = c.filters(heavy=False) + ["", "a/#/b", "a+", "#/x", "#", "+", "+/+", "+/#", "$c/#", "$c/+", "$nope/#", "+/+/+/+"]
    for _ in range(k):
        r = rng.random()
        if r < 0.3:
            fs.append(rand_filter(rng, 6))
        elif r < 0.5:
            fs.append("/".join("+" if rng.random() < 0.6 else t for t in rand_topic(rng, 5).split("/")))
        elif r < 0.6:
            fs.append("$" + rand_topic(rng, 4))
        else:
            fs.append(rng.choice(c.filters(heavy=False)))
    return fs


def _lists(rt, filters):
    w = rt.match_batch(*R.pack(filters))
    o = w["offsets"]
    return [None if w["counts"][i] < 0 else sorted(int(x) for x in w["ids"][o[i]:o[i + 1]]) for i in range(len(filters))]


@pytest.fixture(scope="module")
def corpus():
    c = R.retained_edge_corpus()
    eng, rt = _load(c, "bulk"), c.load_oracle(orc)
    yield c, eng, rt
    eng.close()


@pytest.mark.parametrize("max_batch,wait_us,producers", [(1, 0, 1), (64, 200, 4), (4096, 500, 2)])
def test_retained_batcher_delivers_every_filter_once_with_the_oracle_list(corpus, max_batch, wait_us, producers):
    c, eng, rt = corpus
    rng = random.Random(max_batch)
    filters = _filters(rng, c, 1500)
    want = _lists(rt, filters)
    got, lock = {}, threading.Lock()

    @N.GM_MATCH_CB
    def cb(user, cookie, status, ids, n_ids):
        lst = sorted(ids[i] for i in range(n_ids)) if status == 0 else ("invalid" if status == N.GM_ERR_INVALID_TOPIC else status)
        with lock:
            assert cookie not in got
            got[cookie] = lst

    cfg = N.GmBatcherConfig(C.sizeof(N.GmBatcherConfig), max_batch, wait_us, 2, cb, None)
    h = C.c_void_p()
    lib = N.lib()
    assert lib.gm_retain_batcher_create(eng._h, C.byref(cfg), C.byref(h)) == 0
    pkt = (C.c_uint8 * 7).from_buffer_copy(b"\x30\x05\x00\x03a/b")
    assert lib.gm_submit_publish(h, pkt, 7, 10 ** 9) == N.GM_ERR_INVALID_ARG     # a PUBLISH topic is not a filter

    def produce(k):
        for i in range(k, len(filters), producers):
            b = filters[i].encode()
            assert lib.gm_submit(h, b, len(b), i) == 0

    ths = [threading.Thread(target=produce, args=(k,)) for k in range(producers)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert lib.gm_batcher_drain(h) == 0
    lib.gm_batcher_destroy(h)
    assert len(got) == len(filters)
    for i, f in enumerate(filters):
        assert got[i] == (want[i] if want[i] is not None else "invalid"), f


def _both_paths(eng, rt, filters, what):
    """gm_retain_match_batch with small_graphs 1 and 0: identical spans and id multisets, equal to the oracle's"""
    fb, fo = R.pack(filters)
    w = _canon(rt.match_batch(fb, fo))
    need = int(w[0].clip(0).sum())
    out = []
    for graphs in (1, 0):
        eng.debug_knob("small_graphs", graphs)
        rc, needed, res = _host(eng, fb, fo, need)
        assert rc == N.GM_OK and needed == need, (what, graphs, rc, needed, need)
        _same(res, w, f"{what} (small_graphs {graphs})")
        out.append(res)
    eng.debug_knob("small_graphs", 1)
    assert (out[0].spans == out[1].spans).all(), f"{what}: spans differ between the graph and the pipelined path"
    return w


SIZES = (1, 7, 64, 65, 2048, 2049)


def test_graph_path_equals_pipelined_path_at_the_tier_edges(corpus):
    c, eng, rt = corpus
    rng = random.Random(3)
    pool = _filters(rng, c, 2100)
    for n in SIZES:
        _both_paths(eng, rt, pool[:n], f"{n} filters")
        _both_paths(eng, rt, c.batch(n), f"corpus batch of {n}")


def test_graph_path_follows_mutations_flushes_and_compaction():
    """Rounds that deepen the tree, add a `$` root, put a `$` root first in the root order, and compact: every round's
    lookups through both paths, so a graph that is not re-captured after a flush (view_epoch) answers from a stale view."""
    c = R.retained_edge_corpus()
    eng, rt = _load(c, "bulk"), c.load_oracle(orc)
    rng = random.Random(11)
    probe = _filters(rng, c, 300) + ["dp/#", "dp/+/+/#", "$z/#", "$z/+", "#", "+/+"]
    try:
        for rnd in range(4):
            for n in (1, 7, 64, 65):
                _both_paths(eng, rt, probe[-n:] if n < 10 else probe[:n], f"round {rnd}: {n} filters")
            if rnd == 0:                                     # deepen the tree: more rounds in the graph
                t = "dp/" + "/".join(["d"] * 18)
            elif rnd == 1:                                   # a new `$` root
                t = "$z/a/b"
            else:                                            # a `$` root ahead of the plain ones, then a compaction
                t = "$a/x"
            eng.retain_set(t, 900_000 + rnd)
            rt.insert(t, 900_000 + rnd)
            if rnd == 3:
                eng.compact()
            for k in range(20):
                t = rand_topic(rng, 7)
                try:
                    eng.retain_set(t, 910_000 + rnd * 100 + k)
                except Exception:
                    continue
                rt.remove(t)
                rt.insert(t, 910_000 + rnd * 100 + k)
        _both_paths(eng, rt, probe[:2048], "after the rounds: 2048 filters")
    finally:
        eng.close()


TIER0_IDS = 4096              # engine.cu small_graph_new: ids the 64-filter tier holds


def _launches(eng, fn):
    l0 = eng.kernel_launches()
    r = fn()
    return r, eng.kernel_launches() - l0


def _one_attempt(eng, fb, fo, need):
    """kernel launches of one pipelined attempt (small_graphs 0, the default scratch)"""
    eng.debug_knob("small_graphs", 0)
    _, one = _launches(eng, lambda: _host(eng, fb, fo, need))
    eng.debug_knob("small_graphs", 1)
    return one


def test_small_batch_beyond_the_tier_id_capacity_and_the_exact_capacity_edge(corpus):
    """A one-filter `#` (tens of thousands of handles, more than the tier holds) falls back with the same results; on the
    graph path cap = needed succeeds and needed - 1 is GM_ERR_CAPACITY reporting `needed`, answered by the graph alone."""
    c, eng, rt = corpus
    for filters in (["#"], ["w/#"], ["w/k257/#", "pi/+"]):
        _both_paths(eng, rt, filters, f"{filters} beyond the tier")
    checked = 0
    for filters in (["pi/+/k", "a/#/b"], ["w/k9/+"], ["pi/+"], ["w/k513/+/zz", "pi/+"], c.filters(heavy=False)[:8]):
        fb, fo = R.pack(filters)
        w = _canon(rt.match_batch(fb, fo))
        need = int(w[0].clip(0).sum())
        if not 0 < need <= TIER0_IDS:
            continue
        one = _one_attempt(eng, fb, fo, need)
        (rc, needed, res), n_l = _launches(eng, lambda: _host(eng, fb, fo, need))
        assert rc == N.GM_OK and needed == need and n_l == one, (filters, rc, needed, need, n_l, one)
        _same(res, w, f"{filters[0]} cap = needed")
        (rc, needed, _), n_l = _launches(eng, lambda: _host(eng, fb, fo, need - 1))
        assert rc == N.GM_ERR_CAPACITY and needed == need and n_l == one, (filters, rc, needed, need, n_l, one)
        checked += 1
    assert checked >= 2


def test_graph_overflow_falls_back_grows_and_the_next_call_recaptures(corpus):
    """From retain_caps 64 the graph's frontier overflows: the call falls back, the pipelined path grows the scratch, and
    the next small call re-captures with the grown scratch and runs as one graph launch."""
    c, eng, rt = corpus
    checked = 0
    try:
        for filters in (["w/k513/+/zz"], ["pi/+"], ["pi/+/k", "w/k513/+/zz"], c.filters(heavy=False)[:8]):
            fb, fo = R.pack(filters)
            w = _canon(rt.match_batch(fb, fo))
            need = int(w[0].clip(0).sum())
            if need > TIER0_IDS:
                continue
            eng.debug_knob("retain_caps", 1 << 22)
            _both_paths(eng, rt, filters, f"{filters[0]} default scratch")
            one = _one_attempt(eng, fb, fo, need)
            eng.debug_knob("retain_caps", R.RQ)
            (rc, needed, res), n_l = _launches(eng, lambda: _host(eng, fb, fo, need))
            assert rc == N.GM_OK and needed == need
            _same(res, w, f"{filters[0]} from 64 entries")
            assert n_l >= 3 * one, (filters, n_l, one)                 # the graph + at least two pipelined attempts
            (rc, needed, res), n_l = _launches(eng, lambda: _host(eng, fb, fo, need))
            assert rc == N.GM_OK and needed == need
            _same(res, w, f"{filters[0]} after the growth")
            assert n_l == one, f"{filters}: the next small call did not run as one re-captured graph ({n_l} launches, one attempt = {one})"
            checked += 1
    finally:
        eng.debug_knob("retain_caps", 1 << 22)
    assert checked >= 3


def test_retained_and_match_batchers_on_one_engine_at_the_same_time():
    c = R.retained_edge_corpus()
    eng, rt = _load(c, "bulk"), c.load_oracle(orc)
    rng = random.Random(21)
    tree = orc.TopicTree()
    for i in range(2000):
        f = rand_filter(rng, 5)
        try:
            eng.add(f, i)
        except Exception:
            continue
        tree.insert(f, i)
    filters = _filters(rng, c, 1200)
    topics = [rand_topic(rng, 6) for _ in range(1500)]
    want_r = _lists(rt, filters)
    got = {"r": {}, "m": {}}
    lock = threading.Lock()

    def make_cb(kind):
        @N.GM_MATCH_CB
        def cb(user, cookie, status, ids, n_ids):
            with lock:
                got[kind][cookie] = sorted(ids[i] for i in range(n_ids)) if status == 0 else None
        return cb

    cbs = {k: make_cb(k) for k in "rm"}
    lib = N.lib()
    hs = {}
    for k, create in (("r", lib.gm_retain_batcher_create), ("m", lib.gm_batcher_create)):
        cfg = N.GmBatcherConfig(C.sizeof(N.GmBatcherConfig), 64, 200, 2, cbs[k], None)
        hs[k] = C.c_void_p()
        assert create(eng._h, C.byref(cfg), C.byref(hs[k])) == 0

    def produce(k, items, part):
        for i in range(part, len(items), 2):
            b = items[i].encode()
            assert lib.gm_submit(hs[k], b, len(b), i) == 0

    ths = [threading.Thread(target=produce, args=(k, items, p)) for k, items in (("r", filters), ("m", topics)) for p in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    for h in hs.values():
        assert lib.gm_batcher_drain(h) == 0
        lib.gm_batcher_destroy(h)
    try:
        assert len(got["r"]) == len(filters) and len(got["m"]) == len(topics)
        for i, f in enumerate(filters):
            assert got["r"][i] == want_r[i], f
        for i, t in enumerate(topics):
            w = tree.matches(t)
            assert got["m"][i] == (sorted(w) if w is not None else None), t
    finally:
        eng.close()


def test_retained_latency_probe_reports_sane_numbers(corpus):
    c, eng, rt = corpus
    fb, fo = R.pack(c.filters(heavy=False))
    lat = N.GmLatency()
    for burst, rounds in ((1, 200), (64, 20)):
        assert N.lib().gm_retain_batcher_probe(eng._h, fb.ctypes.data, fo.ctypes.data, len(fo) - 1, burst, rounds, 0, C.byref(lat)) == 0
        d = lat.as_dict()
        assert d["samples"] == burst * rounds and 0 < d["p50_us"] <= d["p99_us"] <= d["max_us"] < 5e6 and d["topics_per_s"] > 0
