"""GPU tier: every match and retained-lookup entry point sees ONE whole flushed state while the writer script of
tests/_flush_script.py mutates, flushes and compacts beside it.

Nine reader threads call the engine (ctypes releases the GIL, so the calls overlap the writer and each other) and only
record (before, after, result); everything is checked after the join: each call against the states its window allows
(`_flush_script.check`), with GM_FLAG_MANUAL_FLUSH only the flushed ones.  The script grows the edge table and the
dictionary, compacts the value sets, raises max_depth past 8 and lowers it with gm_compact, creates extra tree 1 and
gives the first retained deadline while the readers run."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest
import torch

from rmqtt_b200 import _native as N
from rmqtt_b200.engine import Engine, GpuMqttError

import _flush_script as S

pytestmark = pytest.mark.gpu

WRITER_TIMEOUT_S, READER_TIMEOUT_S = 600, 120


@pytest.fixture(scope="module")
def fx():
    bg = S.Background()
    ops = S.script()
    return bg, ops, S.Model(ops, bg)


def _batches(bg):
    """The readers' batches; probe keys are ("sub", tree, topic) and ("ret", now, filter)"""
    sub = lambda t, tr=0: (t, tr, ("sub", tr, t))
    ret = lambda f, now=S.NOW: (f, 0, ("ret", now, f))
    bt = lambda i, tr=0: (bg.topics[i % len(bg.topics)], tr, bg.topic_want[i % len(bg.topics)] if tr == 0 else ())
    bf = lambda i: (bg.filters[i], 0, bg.filter_want[i])
    inv_t = [(t, 0, None) for t in S.INVALID_TOPICS]
    inv_f = [(f, 0, None) for f in S.INVALID_FILTERS]
    probes = [sub(t) for t in S.SUB_PROBES]
    b = {}
    # R1: the tier-0 graph (<= 64 rows, <= 4096 ids): a few probes, each matching up to W values of w/#
    b["R1"] = S.Batch([sub(t) for t in S.SUB_PROBES[:6]] + inv_t + [bt(i) for i in range(56)])
    b["R2"] = S.Batch(probes + inv_t + [bt(i) for i in range(1500 - len(probes) - 2)])                 # tier-1 graph
    # R3: 20 K rows in chunks of 1024, probes in every chunk
    rows = []
    for c in range(20):
        rows += [sub(S.SUB_PROBES[(3 * c + k) % len(S.SUB_PROBES)]) for k in range(3)] + [bt(i) for i in range(c * 1000, c * 1000 + 1021)]
    b["R3"] = S.Batch(rows[:19_997] + inv_t + [sub("w/x")])
    b["R4"] = S.Batch(probes + inv_t + [bt(i) for i in range(2000, 2060)])
    b["R5"] = S.Batch(probes + inv_t + [bt(i) for i in range(3000, 3200)])
    small = [ret(f) for f in S.RET_PROBES[:12]] + inv_f
    b["R6s"] = S.Batch(small + [bf(i) for i in range(40 - len(small))])
    rp = [ret(f) for f in S.RET_PROBES + S.RET_BIG_PROBES]
    b["R6l"] = S.Batch(rp + inv_f + [bf(i) for i in range(3000 - len(rp) - 2)])
    b["R7"] = S.Batch(rp + inv_f + [bf(i) for i in range(200)])
    b["R8"] = S.Batch([sub(t) for t in S.SUB_PROBES[:10]] + [sub(t, 1) for t in S.TREE_PROBES] + inv_t +
                      [bt(i, 1) for i in range(4000, 4040)] + [bt(i) for i in range(4040, 4080)])
    return b


def _epoch(lib, h):
    v = N.GmValues()
    assert lib.gm_values_view(h, C.byref(v)) == 0
    return int(v.epoch)


def _run(manual, bg, ops, model):
    os.environ["GM_WIN_MIN_SLOTS_LOG2"] = "3"
    try:
        eng = Engine(manual_flush=manual)
    finally:
        os.environ.pop("GM_WIN_MIN_SLOTS_LOG2", None)
    lib = N.lib()
    bg.load(eng)
    eng.debug_knob("e2e_chunk", 1024)
    batches = _batches(bg)
    prog = S.Progress()
    done = threading.Event()
    rec = {k: [] for k in ("R1", "R2", "R3", "R4", "R5", "R6", "R7", "R8", "R9p", "R9r")}
    skipped = {"R4": 0}
    errors = []
    stats = []

    def loop(name, call):
        def body():
            try:
                while not done.is_set():
                    before = prog.before()
                    res = call()
                    if res is not None:
                        rec[name].append((before, prog.after(), res))
            except Exception as ex:          # noqa: BLE001
                errors.append((name, repr(ex)))
        return body

    def host(name, fn):
        bt = batches[name]
        return lambda: (bt, S.canonical_lists(*_raw(fn(bt))))

    def _raw(res):
        return res.spans, res.ids, res.status

    def r4():
        bt = batches["R4"]
        e0 = _epoch(lib, eng._h)
        spans, descs, status, _ = eng.match_batch_desc(bt.blob, bt.offs)
        try:
            ids = eng.desc_expand(descs) if len(descs) else np.zeros(0, np.uint32)
        except GpuMqttError:
            ids = None
        if _epoch(lib, eng._h) != e0:
            skipped["R4"] += 1
            return None
        assert ids is not None, "descriptors of an unchanged epoch could not be expanded"
        cnt = descs[:, 1].astype(np.int64)
        assert (cnt != 0xFFFF).all()            # (no value set of this workload reaches the indirect form)
        dstart = np.zeros(len(cnt) + 1, np.int64)
        np.cumsum(cnt, out=dstart[1:])
        d0 = spans[:, 0].astype(np.int64)
        d1 = d0 + spans[:, 1].astype(np.int64)
        ispans = np.stack([dstart[d0], dstart[d1] - dstart[d0]], axis=1)
        return bt, S.canonical_lists(ispans, ids, status)

    dev = torch.device("cuda")

    def device_reader(name, retained):
        bt = batches[name]
        stream = torch.cuda.Stream()
        n = len(bt.rows)
        cap = 1 << 20
        with torch.cuda.stream(stream):
            d_blob = torch.from_numpy(np.concatenate([bt.blob, np.zeros(16, np.uint8)])).to(dev)
            d_offs = torch.from_numpy(bt.offs.view(np.int32)).to(dev)
            d_spans = torch.zeros((n, 2), dtype=torch.int32, device=dev)
            d_ids = torch.zeros(cap, dtype=torch.int32, device=dev)
            d_status = torch.zeros(n, dtype=torch.int32, device=dev)
            d_needed = torch.zeros(1, dtype=torch.int64, device=dev)
        stream.synchronize()

        def call():
            with torch.cuda.stream(stream):
                if retained:
                    needed = C.c_uint64(0)
                    rc = lib.gm_retain_match_batch_device_at(eng._h, S.NOW, d_blob.data_ptr(), len(bt.blob), d_offs.data_ptr(), n, d_spans.data_ptr(),
                                                             d_ids.data_ptr(), cap, C.byref(needed), d_status.data_ptr(), stream.cuda_stream)
                    assert rc == 0, rc
                    m = int(needed.value)
                else:
                    eng.match_batch_device(d_blob, d_offs, d_spans, d_ids, d_needed, d_status, stream.cuda_stream)
                    m = int(d_needed.item())
                assert m <= cap
                out = (d_spans.cpu().numpy().view(np.uint32), d_ids[:m].cpu().numpy().view(np.uint32), d_status.cpu().numpy())
            return bt, S.canonical_lists(*out)
        return call

    r6_turn = [0]

    def r6():
        r6_turn[0] += 1
        bt = batches["R6s" if r6_turn[0] % 2 else "R6l"]
        return bt, S.canonical_lists(*_raw(eng.retain_match_batch(bt.blob, bt.offs, now_ms=S.NOW)))

    # R9: one producer per batcher; each callback is checked against its own submit -> callback window
    cb_lock = threading.Lock()
    pending = {}

    def make_cb(name):
        @N.GM_MATCH_CB
        def cb(user, cookie, status, ids, n_ids):
            lst = tuple(sorted(ids[i] for i in range(n_ids))) if status == 0 else None
            after = prog.after()
            with cb_lock:
                key, before = pending.pop(cookie)
                rec[name].append((before, after, (key, status, lst)))
        return cb

    cbs = {"R9p": make_cb("R9p"), "R9r": make_cb("R9r")}
    handles = {}
    for name, create in (("R9p", lib.gm_batcher_create), ("R9r", lib.gm_retain_batcher_create)):
        cfg = N.GmBatcherConfig(C.sizeof(N.GmBatcherConfig), 64, 200, 2, cbs[name], None)
        h = C.c_void_p()
        assert create(eng._h, C.byref(cfg), C.byref(h)) == 0
        handles[name] = h
    cookie = [0]

    def producer(name, keys):
        h = handles[name]

        def call():
            for key in keys:
                with cb_lock:
                    cookie[0] += 1
                    c = cookie[0]
                    pending[c] = (key, prog.before())
                b = key[2].encode()
                assert lib.gm_submit(h, b, len(b), c) == 0
            assert lib.gm_batcher_drain(h) == 0
            return None
        return call

    readers = {
        "R1": host("R1", lambda bt: eng.match_batch(bt.blob, bt.offs)),
        "R2": host("R2", lambda bt: eng.match_batch(bt.blob, bt.offs)),
        "R3": host("R3", lambda bt: eng.match_batch(bt.blob, bt.offs)),
        "R4": r4,
        "R5": device_reader("R5", False),
        "R6": r6,
        "R7": device_reader("R7", True),
        "R8": host("R8", lambda bt: eng.match_batch_trees(bt.blob, bt.offs, bt.trees)),
        "R9p": producer("R9p", [("sub", 0, t) for t in S.SUB_PROBES]),
        "R9r": producer("R9r", [("ret", S.LATE, f) for f in S.RET_PROBES + S.RET_BIG_PROBES]),
    }

    def on_flush():
        stats.append((eng.stats(), _epoch(lib, eng._h)))

    start = (eng.stats(), _epoch(lib, eng._h))

    def writer():
        try:
            S.run_writer(eng, ops, prog, on_flush)
        except Exception as ex:              # noqa: BLE001
            errors.append(("writer", repr(ex)))
        finally:
            done.set()

    t0 = time.time()
    ths = [threading.Thread(target=loop(k, f), daemon=True, name=k) for k, f in readers.items()]
    wt = threading.Thread(target=writer, daemon=True, name="writer")
    for t in ths:
        t.start()
    wt.start()
    wt.join(WRITER_TIMEOUT_S)
    assert not wt.is_alive(), "the writer did not finish"
    for t in ths:
        t.join(READER_TIMEOUT_S)
    assert not [t.name for t in ths if t.is_alive()], "reader threads did not finish"
    elapsed = time.time() - t0
    assert not errors, errors
    for h in handles.values():
        lib.gm_batcher_destroy(h)
    assert not pending

    # ---- every recorded call ----
    report = {}
    for name, calls in rec.items():
        seen, spanning = set(), 0
        for before, after, res in calls:
            lo, hi = S.window(before, after, manual)
            if name.startswith("R9"):
                key, status, lst = res
                assert status == 0, (name, key, status)
                st = model.states({key: lst}, lo, hi, manual)
                assert len(st), f"{name} {key}: no legal state in [{lo}, {hi}]: " + S.describe(model, {key: lst}, lo, hi, manual)
            else:
                bt, out = res
                try:
                    st = S.check(model, bt, *out, lo, hi, manual)
                except AssertionError as ex:
                    raise AssertionError(f"{name}, window [{lo}, {hi}]: {ex}") from None
            seen.add(int(st[0]))
            spanning += S.spans_flush(before, after)
        report[name] = (len(calls), len(seen), spanning)
    kind = "manual flush" if manual else "automatic flush"
    print(f"\n{kind}: writer + readers {elapsed:.1f} s, {model.n} mutations, {prog.flushes_done} flushes")
    for name, (calls, seen, spanning) in report.items():
        extra = f", {skipped['R4']} skipped (epoch moved)" if name == "R4" else ""
        print(f"  {name}: {calls} calls, {seen} distinct states, {spanning} spanning a flush{extra}")
    assert all(report[k][0] > 0 for k in report), report
    assert report["R4"][0] > 0
    assert sum(r[2] for r in report.values()) > 0, "no call overlapped a flush"
    # the first deadline appeared while the retained readers ran: calls on both sides of it
    for name in ("R6", "R7"):
        his = [S.window(b, a, manual) for b, a, _ in rec[name]]
        assert any(h < model.first_deadline for _, h in his) and any(l >= model.first_deadline for l, _ in his), name

    # ---- coverage: what the writer made the flushes ship ----
    st0, e0 = start
    assert max(s["edge_slots"] for s, _ in stats) > st0["edge_slots"]
    assert max(s["dict_slots"] for s, _ in stats) > st0["dict_slots"]
    epochs = [e0] + [e for _, e in stats]
    assert sum(1 for a, b in zip(epochs, epochs[1:]) if b != a) >= 3 and epochs == sorted(epochs)
    depth = [s["max_depth"] for s, _ in stats]
    assert max(depth) > 8 and depth[-1] <= 8

    # ---- after the join: every entry point once, sequentially, against the final state ----
    eng.flush()
    n = model.n
    final = {k: f for k, f in readers.items() if not k.startswith("R9")}
    for name, call in list(final.items()) + [("R6", r6)]:          # (R6 twice: its small and its large batch)
        bt, out = call()
        S.check(model, bt, *out, n, n, manual)
    for name, keys in (("R9p", [("sub", 0, t) for t in S.SUB_PROBES]), ("R9r", [("ret", S.LATE, f) for f in S.RET_PROBES + S.RET_BIG_PROBES])):
        for key in keys:
            got = eng.matches(key[2]) if name == "R9p" else eng.retain_matches(key[2])
            assert tuple(got) == model.expected(key, n), key
    eng.close()


@pytest.mark.parametrize("manual", [False, True], ids=["auto_flush", "manual_flush"])
def test_every_entry_point_sees_one_flushed_state_under_concurrent_flushes(manual, fx):
    _run(manual, *fx)
