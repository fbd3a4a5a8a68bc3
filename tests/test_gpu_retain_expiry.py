"""GPU tier: expiry of retained messages on the device — gm_retain_match_batch_at through the small-graph path (up to 2048
filters, at the tier edges) and the pipelined path against tests/_retain_expiry.py's restatement of the reference, the
capacity protocol, the device entry point and the retained batcher against the wall clock, seeded rounds of set / set_ttl /
remove / sweep / flush, and an engine without deadlines launching what it launched before."""
import ctypes as C
import random
import threading

import numpy as np
import pytest
import torch

from _retain_expiry import TimedRetain
from oracle import oracle as orc
from rmqtt_b200 import _native as N
from rmqtt_b200 import workload as wl
from rmqtt_b200.engine import Engine, MatchResult, _vp, pack
from test_gpu_edges import _to_dev

pytestmark = pytest.mark.gpu

NOW = 1_760_000_000_000
FAR = 1 << 62                      # a deadline far in the future


def _at(eng, fb, fo, now, cap, ids=None):
    """gm_retain_match_batch_at with an exact capacity -> (rc, needed, MatchResult or None, the output array)"""
    n = len(fo) - 1
    spans, status = np.zeros((n, 2), dtype=np.uint32), np.zeros(n, dtype=np.int32)
    ids = np.zeros(max(cap, 1), dtype=np.uint32) if ids is None else ids
    needed = C.c_uint64(0)
    rc = eng._lib.gm_retain_match_batch_at(eng._h, now, _vp(fb), _vp(fo), n, _vp(spans), _vp(ids), cap, C.byref(needed), _vp(status))
    return rc, int(needed.value), (MatchResult(spans, ids[:int(needed.value)], status, int(needed.value)) if rc == N.GM_OK else None), ids


def _want(rt, dl_arr, fb, fo, now):
    """the oracle's lists without the handles expired at `now` (dl_arr: deadline per handle, ~0 = none) -> (counts, sorted ids)"""
    w = rt.match_batch(fb, fo)
    counts, o, ids = w["counts"].copy(), w["offsets"].astype(np.int64), w["ids"]
    live = dl_arr[ids] > np.uint64(now)
    out = []
    for i in range(len(counts)):
        seg = ids[o[i]:o[i + 1]][live[o[i]:o[i + 1]]]
        if counts[i] >= 0:
            counts[i] = len(seg)
        out.append(np.sort(seg))
    return counts, (np.concatenate(out) if out else np.zeros(0, np.uint32)).astype(np.uint32)


def _same(res, want, what):
    counts, ids = res.canonical()
    assert (counts == want[0]).all(), f"{what}: counts differ at {np.nonzero(counts != want[0])[0][:5]}"
    assert len(ids) == len(want[1]) and (ids == want[1]).all(), what


@pytest.fixture(scope="module")
def c4():
    """C4's retained topics and filters, scaled to 300 K topics: 30 % carry deadlines around NOW, some exactly at NOW"""
    blob, offs, vals = wl.gen_retained(wl.C4, 300_000)
    fb, fo = wl.gen_retain_filters(wl.C4, 4096)
    rng = np.random.default_rng(7)
    dl = np.zeros(len(vals), np.uint64)
    has = rng.random(len(vals)) < 0.3
    dl[has] = (NOW + rng.integers(-3, 4, has.sum())).astype(np.uint64)
    eng = Engine(device=0)
    assert eng.retain_bulk_load(blob, offs, vals, dl) == len(vals)
    rt = orc.RetainTree()
    rt.bulk_insert(blob, offs, vals)
    dl_arr = np.where(dl == 0, np.uint64(0xFFFFFFFFFFFFFFFF), dl)
    yield eng, rt, dl_arr, fb, fo
    eng.close()


def _sub(fb, fo, a, b):
    o = fo[a:b + 1].astype(np.int64)
    return fb[o[0]:o[-1]].copy(), (o - o[0]).astype(np.uint32)


@pytest.mark.parametrize("graphs", [1, 0])
def test_c4_scaled_lookups_at_several_nows_equal_the_reference(c4, graphs):
    eng, rt, dl_arr, fb, fo = c4
    eng.debug_knob("small_graphs", graphs)
    try:
        for n in (1, 64, 65, 2048) + ((4096,) if not graphs else ()):
            sb, so = _sub(fb, fo, 0, n)
            for now in (NOW - 4, NOW - 1, NOW, NOW + 1, NOW + 4):
                want = _want(rt, dl_arr, sb, so, now)
                need = int(want[0].clip(0).sum())
                rc, needed, res, _ = _at(eng, sb, so, now, need)
                assert rc == N.GM_OK and needed == need, (n, now, rc, needed, need)
                _same(res, want, f"{n} filters, now {now - NOW:+d}, small_graphs {graphs}")
    finally:
        eng.debug_knob("small_graphs", 1)


@pytest.mark.parametrize("graphs", [1, 0])
def test_capacity_protocol_counts_live_handles_and_leaves_the_rest_untouched(c4, graphs):
    eng, rt, dl_arr, fb, fo = c4
    eng.debug_knob("small_graphs", graphs)
    try:
        sb, so = _sub(fb, fo, 0, 64)
        want = _want(rt, dl_arr, sb, so, NOW)
        live = int(want[0].clip(0).sum())
        assert live > 0
        ids = np.full(live + 64, 0xEEEEEEEE, dtype=np.uint32)
        rc, needed, _, _ = _at(eng, sb, so, NOW, live - 1, ids)
        assert rc == N.GM_ERR_CAPACITY and needed == live
        ids[:] = 0xEEEEEEEE
        rc, needed, res, ids = _at(eng, sb, so, NOW, live, ids)
        assert rc == N.GM_OK and needed == live
        _same(res, want, f"exact capacity, small_graphs {graphs}")
        assert (ids[live:] == 0xEEEEEEEE).all()
    finally:
        eng.debug_knob("small_graphs", 1)


def _wall_engine():
    eng, ref = Engine(device=0), TimedRetain(orc)
    for i in range(400):
        d = (1, FAR, 0)[i % 3]                     # long expired, far in the future, none
        eng.retain_set(f"w/{i % 20}/{i}", 1000 + i, deadline_ms=d)
        ref.set_with_timeout(f"w/{i % 20}/{i}", 1000 + i, d)
    return eng, ref


def test_device_entry_point_and_plain_call_use_the_wall_clock():
    eng, ref = _wall_engine()
    filters = ["w/#", "w/+/+", "#", "w/3/+", "w/7/#", "w/1/1001", "w/2/1002"]
    fb, fo = pack(filters)
    want = [ref.get_message(f, NOW) for f in filters]
    res = eng.retain_match_batch(fb, fo)
    assert [res.sorted_list(i) for i in range(len(filters))] == want
    n = len(filters)
    d_blob, d_offs = _to_dev(fb, fo)
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    d_ids = torch.full((4096,), -1, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    needed = eng.retain_match_batch_device(d_blob, d_offs, d_spans, d_ids, d_status, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    spans, ids = d_spans.cpu().numpy().astype(np.uint32), d_ids.cpu().numpy().astype(np.uint32)
    assert needed == sum(len(w) for w in want)
    for i in range(n):
        assert sorted(ids[spans[i, 0]:spans[i, 0] + spans[i, 1]].tolist()) == want[i], filters[i]
    eng.close()


def test_retained_batcher_uses_the_wall_clock():
    eng, ref = _wall_engine()
    filters = [f"w/{k}/+" for k in range(20)] + ["w/#", "#"]
    got, lock = {}, threading.Lock()

    @N.GM_MATCH_CB
    def cb(user, cookie, status, ids, n_ids):
        with lock:
            got[cookie] = sorted(ids[i] for i in range(n_ids)) if status == 0 else status

    cfg = N.GmBatcherConfig(C.sizeof(N.GmBatcherConfig), 8, 100, 2, cb, None)
    h = C.c_void_p()
    lib = N.lib()
    assert lib.gm_retain_batcher_create(eng._h, C.byref(cfg), C.byref(h)) == 0
    for i, f in enumerate(filters):
        b = f.encode()
        assert lib.gm_submit(h, b, len(b), i) == 0
    assert lib.gm_batcher_drain(h) == 0
    lib.gm_batcher_destroy(h)
    for i, f in enumerate(filters):
        assert got[i] == ref.get_message(f, NOW), f
    eng.close()


def test_seeded_rounds_of_set_set_ttl_remove_sweep_and_flush():
    rng = random.Random(31)
    eng, ref = Engine(device=0, manual_flush=True), TimedRetain(orc)
    now = NOW
    filters = ["#", "r/#", "r/+/+", "r/+/3", "+/#", "r/5/#"]
    fb, fo = pack(filters)
    for rnd in range(12):
        for _ in range(300):
            t = f"r/{rng.randrange(12)}/{rng.randrange(12)}"
            op = rng.random()
            if op < 0.55:
                h = rng.randrange(1, 3000)
                if any(hh == h and tt != t for tt, hh in ref.val.items()):
                    continue                                  # every handle stays under one topic
                d = rng.choice([0, now + rng.randrange(-20, 60), now])
                eng.retain_set(t, h, deadline_ms=d)
                ref.set_with_timeout(t, h, d)
            elif op < 0.8:
                assert eng.retain_remove(t) == ref.remove(t)
            else:
                got = eng.retain_remove_expired(now, rng.choice([1, 5, 1 << 20])).tolist()
                for h in got:
                    assert ref.expired(h, now)
                    ref.remove(next(tt for tt, hh in ref.val.items() if hh == h))
        eng.flush()
        for at in (now - 1, now, now + 30):
            for graphs in (1, 0):
                eng.debug_knob("small_graphs", graphs)
                res = eng.retain_match_batch(fb, fo, now_ms=at)
                assert [res.sorted_list(i) for i in range(len(filters))] == [ref.get_message(f, at) for f in filters], (rnd, at, graphs)
        eng.debug_knob("small_graphs", 1)
        now += 25
    eng.close()


def _launches_and_lists(eng, fb, fo, n_filters):
    out = []
    for graphs in (1, 0):
        eng.debug_knob("small_graphs", graphs)
        l0 = eng.kernel_launches()
        res = eng.retain_match_batch(fb, fo)
        out.append((eng.kernel_launches() - l0, [res.sorted_list(i) for i in range(n_filters)]))
    eng.debug_knob("small_graphs", 1)
    return out


def test_an_engine_without_deadlines_launches_and_returns_what_it_did_before():
    topics = [f"p/{i % 30}/{i}" for i in range(3000)]
    filters = ["#", "p/+/+", "p/3/#", "p/+/17", "+/#"]
    fb, fo = pack(filters)
    plain = Engine(device=0)
    for i, t in enumerate(topics):
        plain.retain_set(t, i)
    base = _launches_and_lists(plain, fb, fo, len(filters))
    touched = Engine(device=0)                                  # the new calls, leaving no deadline behind
    for i, t in enumerate(topics):
        touched.retain_set(t, i, deadline_ms=0 if i % 2 else NOW)
    for i, t in enumerate(topics):
        if i % 2 == 0:
            touched.retain_set(t, i)                            # clears the deadline
    assert touched.retain_remove_expired(FAR, 1 << 20).size == 0
    assert _launches_and_lists(touched, fb, fo, len(filters)) == base
    with_dl = Engine(device=0)                                  # with deadlines: one more kernel (k_retain_live) per launch
    for i, t in enumerate(topics):                              # sequence, the same lists
        with_dl.retain_set(t, i, deadline_ms=FAR if i == 0 else 0)
    got = _launches_and_lists(with_dl, fb, fo, len(filters))
    assert [g[1] for g in got] == [b[1] for b in base]
    per_sequence = 4 + 3 + 1                                    # k_tokenize, k_retain_init, k_retain_scan, k_retain_expand + rounds (depth 3 + 1)
    assert all(b[0] % per_sequence == 0 for b in base)
    assert [g[0] for g in got] == [b[0] + b[0] // per_sequence for b in base]
    for e in (plain, touched, with_dl):
        e.close()
