"""GPU tier of the fast path's id expansion at its tile and capacity edges: the corpus of tests/_tile_edges.py through
gm_match_batch_device (plain and instrumented), gm_match_batch_device_ex (a selection of rows; descriptor mode), the host
entry points (both small-graph tiers, the pipelined path in chunks of 1024 rows) and the one-rank fused gather, at the
default scheduling and with tiles claimed out of order (tile_chunk 7 / 1024, k2_ctas 1 / 3).

Outputs are guarded and patterned as on the CPU tier (tests/test_emu_tile_edges.py, whose checks these are).  Before every
checked call a POISON batch runs on the same engine through the same entry point: ids from values no checked batch yields,
more sets per row; for the device entry points it has as many rows as the checked batch (the same scratch layout, so a
stale tile record or item would point at its ids).  For the host path three poison batches run, each from three threads at
once (so usually on more than one match context; a context none of them leased holds an earlier poison or checked call):
4096 rows through the pipelined path, and one batch that itself runs as each small-graph tier's graph, so that the tier's
own staging holds poison too.  Every result is compared with the oracle, never with another GPU run."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import _tile_edges as T
from rmqtt_b200 import _native as N
from rmqtt_b200.engine import Engine, MatchResult
from test_emu_tile_edges import MP_DIAG_NO_PUBLISH, Guarded, _total, caps_below, check_exact, check_no_publish

pytestmark = pytest.mark.gpu

KNOBS = [{}, {"tile_chunk": 7}, {"tile_chunk": 1024}, {"k2_ctas": 1}, {"k2_ctas": 3}]
DEFAULTS = dict(tile_chunk=1, k2_ctas=0, diag_flags=0, small_graphs=1, e2e_chunk=262144)
DEVICE_SHAPES = [s for s in T.SHAPES if s != "p2049"] + ["p2049"]


class Ctx:
    def __init__(self):
        self.c = T.tile_corpus()
        self.tree = self.c.load_oracle()
        T.check_against_oracle(self.c, self.tree)
        self.eng = Engine(device=0)
        self.c.load_engine(self.eng)
        self.want = {}

    def batch(self, name):
        if name not in self.want:
            tb, to = self.c.packed(name)
            w = self.tree.match_batch(tb, to)
            ids = w["ids"].copy()
            for i in range(len(w["offsets"]) - 1):
                ids[w["offsets"][i]:w["offsets"][i + 1]].sort()
            self.want[name] = (tb, to, w["counts"], ids, w["counters"])
        return self.want[name]

    def poison_for(self, name):
        p = f"{name}#poison"
        if p not in self.c.batches:
            self.c.batches[p] = self.c.poison_batch(len(self.c.batches[name]))
        return p

    def reset(self):
        for k, v in DEFAULTS.items():
            self.eng.debug_knob(k, v)


@pytest.fixture(scope="module")
def gx():
    x = Ctx()
    yield x
    x.eng.close()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class DevGuarded:
    """A Guarded buffer on the device; .host() copies it back into a Guarded for the checks."""

    def __init__(self, n, width, guard, salt):
        self.h = Guarded(n, width, guard, salt)
        self.buf = torch.from_numpy(self.h.buf.view(np.int32)).cuda()
        self.inner = self.buf[guard * width:(guard + n) * width]

    def host(self):
        self.h.buf[:] = self.buf.cpu().numpy().view(np.uint32)
        return self.h


def _blob(tb, to):
    raw = torch.zeros(len(tb) + 64, dtype=torch.uint8, device="cuda")
    base = (16 - raw.data_ptr() % 16) % 16
    d_blob = raw[base:base + len(tb)]
    if len(tb):
        d_blob.copy_(torch.from_numpy(tb))
    return d_blob, torch.from_numpy(to.view(np.int32)).cuda()


def device_call(x, name, cap, *, work=False, desc=False, sel=None, guard=None):
    """gm_match_batch_device(_stats), or gm_match_batch_device_ex with a selection / descriptors -> the emulator-tier tuple"""
    tb, to, counts, _, _ = x.batch(name if sel is None else sel[0])
    n = len(to) - 1 if sel is None else len(sel[1])
    guard = guard if guard is not None else max(_total(x, name), 64) + 1024
    ids = DevGuarded(cap, 2 if desc else 1, guard, 1)
    spans, status = DevGuarded(n, 2, 64, 2), DevGuarded(n, 1, 64, 3)
    d_blob, d_offs = _blob(tb, to)
    d_needed = torch.zeros(1, dtype=torch.int64, device="cuda")
    w = None
    if sel is None and not desc:
        w = x.eng.match_batch_device(d_blob, d_offs, spans.inner, ids.inner, d_needed, status.inner, _stream(), work=work)
    else:
        d_sel = torch.from_numpy(np.asarray(sel[1] if sel else np.arange(n), dtype=np.int32)).cuda()
        out = ids.inner.view(-1, 2) if desc else ids.inner
        w = x.eng.match_batch_device_ex(d_blob, d_offs, spans.inner, out, d_needed, status.inner, _stream(), desc=desc, d_sel=d_sel, n_sel=n, work=work)
    torch.cuda.synchronize()
    rc = 0 if int(d_needed.item()) <= cap else -3
    work4 = np.asarray([w["visited"], w["probed"], w["filters"], w["ids"]], dtype=np.uint64) if w else np.zeros(4, np.uint64)
    return rc, int(d_needed.item()), ids.host(), spans.host(), status.host(), work4, (w or {}).get("deferred", 0)


def poison_device(x, name):
    p = x.poison_for(name)
    check_exact(x, p, device_call(x, p, _total(x, p)), f"poison before {name}")


def check_capacity_dev(x, name, r, cap, what):
    rc, needed, ids, spans, status, _, _ = r
    assert needed == _total(x, name), (what, cap, needed)
    assert ids.guards_intact() and spans.guards_intact() and status.guards_intact(), f"{what}: cap {cap}: written at or past cap"


def check_descriptors(x, name, r, what):
    rc, needed, descs, spans, status, _, _ = r
    cases = x.c.batches[name]
    assert needed == _total(x, name, desc=True) and descs.guards_intact() and spans.guards_intact() and status.guards_intact(), (what, needed)
    sp, d = spans.inner.reshape(-1, 2), descs.inner.reshape(-1, 2)
    assert descs.written(0, needed), f"{what}: a pattern pair is left among the descriptors"
    valid = np.asarray([c.F is not None for c in cases])
    assert (sp[valid, 1] == [c.F for c in cases if c.F is not None]).all(), what
    used = valid & (sp[:, 1] > 0)                   # (an empty span's offset is arbitrary)
    o = np.argsort(sp[used, 0], kind="stable")
    ends = np.cumsum(sp[used, 1][o].astype(np.int64))
    assert (sp[used, 0][o] == ends - sp[used, 1][o]).all() and (ends[-1] if len(ends) else 0) == needed, what
    _, rng, _ = x.eng.values_view()
    cnt = d[:needed, 1].astype(np.int64)
    big = cnt == T.CNT_BIG
    cnt[big] = rng[d[:needed][big, 0], 1]
    starts = np.zeros(needed + 1, dtype=np.int64)
    np.cumsum(cnt, out=starts[1:])
    ids = x.eng.desc_expand(np.ascontiguousarray(d[:needed])) if needed else np.zeros(0, np.uint32)
    d0 = np.where(sp[:, 1] > 0, sp[:, 0], 0).astype(np.int64)
    d1 = d0 + sp[:, 1].astype(np.int64)
    res = MatchResult(np.stack([starts[d0], starts[d1] - starts[d0]], axis=1).astype(np.uint32), ids, status.inner.view(np.int32), len(ids))
    got_c, got_i = res.canonical()
    _, _, counts, wids, _ = x.batch(name)
    assert (got_c == counts).all() and (got_i == wids).all(), f"{what}: expanded descriptors differ"


def _device_shape(x, name, full):
    total = _total(x, name)
    poison_device(x, name)
    check_exact(x, name, device_call(x, name, total), f"{name} device")
    for cap in caps_below(x, name):
        poison_device(x, name)
        check_capacity_dev(x, name, device_call(x, name, cap), cap, f"{name} device")
    poison_device(x, name)
    r = device_call(x, name, total, work=True)
    check_exact(x, name, r, f"{name} instrumented")
    k = x.batch(name)[4]
    assert [int(v) for v in r[5]] == [k["V"], k["E"], k["F"], k["M"]] and r[6] == x.c.n_deferred(name), name
    if not full:
        return
    n = len(x.c.batches[name])
    rows = np.random.default_rng(n).permutation(n)[:max(1, (3 * n) // 4)]
    sname = f"{name}#sel"
    x.c.batches[sname] = [x.c.batches[name][i] for i in rows]
    poison_device(x, name)
    check_exact(x, sname, device_call(x, sname, _total(x, sname), sel=(name, rows)), f"{name} device_ex selection")
    nd = _total(x, name, desc=True)
    poison_device(x, name)
    check_descriptors(x, name, device_call(x, name, nd, desc=True), f"{name} device_ex descriptors")
    if nd:
        poison_device(x, name)
        r = device_call(x, name, nd // 2, desc=True)
        assert r[1] == nd and r[2].guards_intact() and r[3].guards_intact(), f"{name} descriptors at cap {nd // 2}"


@pytest.mark.parametrize("knobs", KNOBS, ids=lambda k: "-".join(f"{a}={b}" for a, b in k.items()) or "defaults")
def test_device_entry_points_on_poisoned_scratch(gx, knobs):
    gx.reset()
    try:
        for k, v in knobs.items():
            gx.eng.debug_knob(k, v)
        for name in DEVICE_SHAPES:
            _device_shape(gx, name, full=not knobs or "tile_chunk" in knobs)
    finally:
        gx.reset()


def test_no_publish_diagnostic_then_exact_again(gx):
    gx.reset()
    for name in ("items65", "holes", "full32", "p2049"):
        poison_device(gx, name)
        gx.eng.debug_knob("diag_flags", MP_DIAG_NO_PUBLISH)
        try:
            r = device_call(gx, name, _total(gx, name))
        finally:
            gx.reset()
        check_no_publish(gx, name, r, f"{name} no-publish")
        poison_device(gx, name)
        check_exact(gx, name, device_call(gx, name, _total(gx, name)), f"{name} after no-publish")


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def host_call(x, name, cap, desc=False):
    """gm_match_batch / gm_match_batch_desc into guarded host buffers"""
    tb, to, _, _, _ = x.batch(name)
    n = len(to) - 1
    ids = Guarded(cap, 2 if desc else 1, max(_total(x, name), 64) + 64, 1)
    spans, status = Guarded(n, 2, 64, 2), Guarded(n, 1, 64, 3)
    needed = C.c_uint64(0)
    fn = x.eng._lib.gm_match_batch_desc if desc else x.eng._lib.gm_match_batch
    rc = fn(x.eng._h, _vp(tb), _vp(to), n, spans.ptr, ids.ptr, cap, C.byref(needed), status.ptr)
    assert rc in (N.GM_OK, N.GM_ERR_CAPACITY), rc
    return (0 if rc == N.GM_OK else -3), int(needed.value), ids, spans, status, np.zeros(4, np.uint64), 0


def poison_host(x):
    """the pipelined path's 4096-row poison batch and each small-graph tier's own, each from three threads at once"""
    for p in ("z4096", "z0_graph", "z1_graph"):
        tb, to, _, _, _ = x.batch(p)
        with ThreadPoolExecutor(3) as ex:
            for res in ex.map(lambda _: x.eng.match_batch(tb, to), range(3)):
                check_exact(x, p, (0, res.needed, _as_guarded(res.ids), _as_guarded(res.spans.reshape(-1)), _as_guarded(res.status.view(np.uint32)), None, 0),
                            "host poison")


def _as_guarded(a):
    g = Guarded(0, 1, 0, 0)
    g.n, g.buf, g.inner, g.fill = len(a), a, a, np.full(len(a), 0xFFFFFFF0, dtype=np.uint32)
    return g


@pytest.mark.parametrize("chunk", [262144, 1024])
def test_host_entry_points_small_graph_tiers_and_pipelined_chunks(gx, chunk):
    gx.reset()
    gx.eng.debug_knob("e2e_chunk", chunk)
    try:
        for name in ("g0_low", "g0_at", "g1_low", "g1_at", "p1", "p33", "items1024", "full32", "step_big", "holes", "p2049"):
            total = _total(gx, name)
            poison_host(gx)
            r = host_call(gx, name, total)
            check_exact(gx, name, r, f"{name} host, chunks of {chunk}")
            for cap in caps_below(gx, name):
                poison_host(gx)
                r = host_call(gx, name, cap)
                assert r[0] == -3, (name, cap)
                check_capacity_dev(gx, name, r, cap, f"{name} host")
            nd = _total(gx, name, desc=True)
            poison_host(gx)
            check_descriptors(gx, name, host_call(gx, name, nd, desc=True), f"{name} host descriptors")
    finally:
        gx.reset()


def _gather(x, name, slab_ids):
    """one step of the fused gather at world 1 into the engine's current block -> (counts, index, spans, ids of the whole slab)"""
    tb, to, _, _, _ = x.batch(name)
    d_blob, d_offs = _blob(tb, to)
    d_status = torch.zeros(len(to) - 1, dtype=torch.int32, device="cuda")
    x.eng.match_gather_device(d_blob, d_offs, d_status, _stream())
    cnt, idx, spans, ids = x.eng.gather_result(_stream())
    return cnt, idx, spans, ids, d_status.cpu().numpy()


def test_one_rank_fused_gather(gx):
    """The GATHER instantiations at world 1, into one block per batch: a poison step (same rows, more ids) fills the slab,
    then the checked step must tile [0, total) with its spans, leave every word past `total` as the poison step left it and
    give the oracle's multisets.  With a slab smaller than the ids, `needed` is exact and the index and span lengths (which
    follow the id slab in the block) are intact."""
    gx.reset()
    for name in ("items1024", "full32", "singles", "holes", "holes_sorted_out", "p65", "p2049"):
        _, to, counts, wids, _ = gx.batch(name)
        n, total = len(to) - 1, _total(gx, name)
        p = gx.poison_for(name)
        for slab in (max(total, _total(gx, p)) + 64, total // 2):
            gx.eng.gather_create(1, 0, n, slab)
            try:
                gx.eng.gather_connect([b"\0" * N.GM_IPC_HANDLE_BYTES])
                _, _, _, before, _ = _gather(gx, p, slab)
                cnt, idx, spans, ids, st = _gather(gx, name, slab)
                assert cnt.tolist() == [[n, total]], (name, slab, cnt.tolist())
                order = np.argsort(idx)
                assert (idx[order] == np.arange(n)).all(), f"{name} gather at slab {slab}: index"
                sp = spans[order]
                assert (sp[st == 0, 1] == counts[st == 0]).all(), f"{name} gather at slab {slab}: span lengths"
                if slab < total:
                    continue
                assert (ids[total:] == before[total:]).all(), f"{name} gather: written past total"
                ok = (st == 0) & (sp[:, 1] > 0)
                off, c = sp[ok, 0].astype(np.int64), sp[ok, 1].astype(np.int64)
                o = np.argsort(off, kind="stable")
                ends = np.cumsum(c[o])
                assert (off[o] == ends - c[o]).all() and (ends[-1] if len(ends) else 0) == total, f"{name} gather: spans do not tile [0, total)"
                got_c, got_i = MatchResult(sp, ids, st, total).canonical()
                assert (got_c == counts).all() and (got_i == wids).all(), f"{name} gather"
            finally:
                gx.eng.gather_destroy()
