"""GPU tier at the size boundaries of the retained lookup: the corpus of tests/_retain_edges.py (child blocks of 8 .. 65537
entries, stage-B survivor lists of 0 / 1 / 255 / 256, the in-place stack and its spill to tasks, parent `#` at every site,
Bloom masks, interleaved `$` roots, the values 0 and 2^32-1, invalid filters, batches of 1 .. 4097 filters) loaded one by one,
in bulk, and in bulk followed by in-place edits — through gm_retain_match_batch and gm_retain_match_batch_device, instrumented
(per-round task counts against the corpus), from a 64-entry scratch, and at the exact capacity edge.  Every answer is
compared with the oracle's RetainTree."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import _retain_edges as R
from oracle import oracle as orc
from rmqtt_b200 import _native as N
from rmqtt_b200.engine import Engine, MatchResult
from test_gpu_edges import _canon, _same, _stream, _to_dev, _vp

pytestmark = pytest.mark.gpu

STATS_RE = re.compile(r"retain stats: .*tasks per round:([ \d]+); descriptors (\d+)")


def _load(c, how):
    """(a) "set": retain_set one by one, the 65537-child node by retain_bulk_load into the non-empty tree; (b) "bulk":
    everything in one retain_bulk_load into the empty tree, down the parallel level-by-level build."""
    eng = Engine(device=0)
    if how == "set":
        for t, v in c.sets:
            eng.retain_set(t, v)
        todo = c.bulk
    else:
        todo = c.all_topics()
    if todo:
        old = {k: os.environ.get(k) for k in ("GM_HOST_PAR_MIN", "GM_HOST_THREADS")}
        os.environ.update(GM_HOST_PAR_MIN="1", GM_HOST_THREADS="4")
        try:
            tb, to = R.pack([t for t, _ in todo])
            assert eng.retain_bulk_load(tb, to, np.asarray([v for _, v in todo], dtype=np.uint32)) == len(todo)
        finally:
            for k, v in old.items():
                os.environ.pop(k) if v is None else os.environ.__setitem__(k, v)
    return eng


def _host(eng, fb, fo, cap):
    """gm_retain_match_batch with an exact capacity -> (rc, needed, MatchResult or None)"""
    n = len(fo) - 1
    spans, status = np.zeros((n, 2), dtype=np.uint32), np.zeros(n, dtype=np.int32)
    ids = np.zeros(max(cap, 1), dtype=np.uint32)
    needed = C.c_uint64(0)
    rc = eng._lib.gm_retain_match_batch(eng._h, _vp(fb), _vp(fo), n, _vp(spans), _vp(ids), cap, C.byref(needed), _vp(status))
    return rc, int(needed.value), (MatchResult(spans, ids, status, int(needed.value)) if rc == N.GM_OK else None)


def _device(eng, fb, fo, cap, shift=0):
    """gm_retain_match_batch_device (torch buffers on the current stream), the blob `shift` bytes past a 16-byte boundary"""
    n = len(fo) - 1
    d_blob, d_offs = _to_dev(fb, fo, shift)
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    d_ids = torch.zeros(cap, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    needed = C.c_uint64(0)
    rc = eng._lib.gm_retain_match_batch_device(eng._h, d_blob.data_ptr(), d_blob.numel(), d_offs.data_ptr(), n, d_spans.data_ptr(),
                                               d_ids.data_ptr() if cap else None, cap, C.byref(needed), d_status.data_ptr(), _stream())
    torch.cuda.synchronize()
    if rc != N.GM_OK:
        return rc, int(needed.value), None
    return rc, int(needed.value), MatchResult(d_spans.cpu().numpy().view(np.uint32), d_ids.cpu().numpy().view(np.uint32),
                                              d_status.cpu().numpy(), int(needed.value))


def _check(eng, rt, filters, what, entry="both", shift=0):
    fb, fo = R.pack(filters)
    w = _canon(rt.match_batch(fb, fo))
    total = int(w[0].clip(0).sum())
    for name, fn in (("host", lambda: _host(eng, fb, fo, total)), ("device", lambda: _device(eng, fb, fo, total, shift))):
        if entry not in ("both", name):
            continue
        rc, needed, res = fn()
        assert rc == N.GM_OK and needed == total, (what, name, rc, needed, total)
        _same(res, w, f"{what} ({name})")
    return w


class Loaded:
    def __init__(self, how):
        self.how = how
        self.c, self.lit = R.retained_edge_corpus(), R.retained_lit_hash_corpus()
        self.rt, self.rt_lit = self.c.load_oracle(orc), self.lit.load_oracle(orc)
        self.eng, self.eng_lit = _load(self.c, how), _load(self.lit, how)

    def pairs(self):
        return ((self.c, self.eng, self.rt), (self.lit, self.eng_lit, self.rt_lit))

    def close(self):
        self.eng.close()
        self.eng_lit.close()


@pytest.fixture(scope="module", params=["set", "bulk"])
def loaded(request):
    x = Loaded(request.param)
    yield x
    x.close()


def test_corpus_through_both_entry_points(loaded):
    """Every filter of both corpora, the batch shapes, and the device entry point with the blob 1 .. 15 bytes off a 16-byte
    boundary; the Bloom-mask and root-order cases proved from the exported image."""
    R.check_constants()
    for c, eng, rt in loaded.pairs():
        _check(eng, rt, c.filters(), f"{loaded.how}: all filters")
        if not c.bulk:
            continue
        img = R.Image(eng.debug_tables()["rnodes"], eng.debug_tables()["rkids"])
        R.bloom_proof(c, img)
        R.root_interleave_proof(c, img)
        for n in R.BATCH_SHAPES:
            _check(eng, rt, c.batch(n), f"{loaded.how}: batch of {n}")
        light = c.filters(heavy=False)
        for shift in range(1, 16):
            _check(eng, rt, light, f"{loaded.how}: blob {shift} bytes past 16", entry="device", shift=shift)


def _stats_line(capfd):
    lines = [m for m in STATS_RE.finditer(capfd.readouterr().err)]
    assert len(lines) == 1, len(lines)
    return [int(x) for x in lines[0].group(1).split()], int(lines[0].group(2))


def test_instrumented_lookups_queue_the_stated_tasks(loaded, capfd):
    """debug_knob("retain_stats", 1): exact results, and the per-round task totals the engine prints equal the corpus's
    stated counts for every shape case, through both entry points."""
    for c, eng, rt in loaded.pairs():
        eng.debug_knob("retain_stats", 1)
        try:
            capfd.readouterr()
            _check(eng, rt, c.filters(), f"{loaded.how}: instrumented, all filters", entry="host")
            _stats_line(capfd)
            for q in c.stated():
                for entry in ("host", "device"):
                    _check(eng, rt, [q.filt], f"{loaded.how}: instrumented {q.filt}", entry=entry)
                    got, _ = _stats_line(capfd)
                    assert got == list(q.tasks) + [0] * (len(got) - len(q.tasks)), (loaded.how, entry, q.filt, got, q.tasks)
        finally:
            eng.debug_knob("retain_stats", 0)


def test_scratch_from_64_entries_grows_each_queue_kind(loaded):
    """From retain_caps 64 (one entry per queue slice): a tasks-only overflow (`w/k513/+/zz`: 3 tasks into one slice, no
    value) and a descriptors-only overflow (`pi/+`: 3 values into one slice, no task) through both entry points, then the
    light filters: exact, and kernel_launches() grew by a whole number of attempts, more than one."""
    c, eng, rt = loaded.c, loaded.eng, loaded.rt
    for filters in (["w/k513/+/zz"], ["pi/+"], c.filters(heavy=False)):
        for entry in ("host", "device"):
            eng.debug_knob("retain_caps", 1 << 22)          # the default size: one attempt
            l0 = eng.kernel_launches()
            _check(eng, rt, filters, f"{filters[0]} default scratch", entry=entry)
            one = eng.kernel_launches() - l0
            eng.debug_knob("retain_caps", R.RQ)
            l0 = eng.kernel_launches()
            _check(eng, rt, filters, f"{filters[0]} from 64 entries", entry=entry)
            grown = eng.kernel_launches() - l0
            assert grown > one and grown % one == 0, (filters[0], entry, grown, one)
    eng.debug_knob("retain_caps", 1 << 22)


def test_capacity_protocol_at_the_exact_edge(loaded):
    """cap_ids = needed succeeds; needed - 1 is GM_ERR_CAPACITY reporting `needed`; cap_ids = 0 on a batch that matches
    nothing (and holds invalid filters) succeeds — on both entry points."""
    c, eng, rt = loaded.c, loaded.eng, loaded.rt
    for filters in (c.batch(1025), ["w/k257/#"], ["pi/+/k", "a/#/b"]):
        fb, fo = R.pack(filters)
        w = _canon(rt.match_batch(fb, fo))
        need = int(w[0].clip(0).sum())
        for fn in (_host, _device):
            rc, needed, res = fn(eng, fb, fo, need)
            assert rc == N.GM_OK and needed == need
            _same(res, w, f"{fn.__name__} cap = needed")
            rc, needed, _ = fn(eng, fb, fo, need - 1)
            assert rc == N.GM_ERR_CAPACITY and needed == need, (fn.__name__, rc, needed, need)
    fb, fo = R.pack(["nope/+", "w/k9/zz/#", "a+", "", "#/x", "s/n0/+/lit"])
    w = _canon(rt.match_batch(fb, fo))
    assert int(w[0].clip(0).sum()) == 0
    for fn in (_host, _device):
        rc, needed, res = fn(eng, fb, fo, 0)
        assert rc == N.GM_OK and needed == 0
        _same(res, w, f"{fn.__name__} cap = 0")


def test_in_place_edits_of_the_bulk_built_image():
    """(c) the bulk-built edge corpus edited in place by the corpus's edit script, each edit checked through both entry points;
    the rstats counters show which edits stayed in place; gm_retain_remove_batch reports 2^32-1 both for a removed value
    2^32-1 and for nothing removed, so only n_removed tells them apart."""
    c = R.retained_edge_corpus()
    eng, rt = _load(c, "bulk"), c.load_oracle(orc)
    _check(eng, rt, ["#"], "first lookup")
    tables = eng.debug_tables()
    proof = R.bloom_proof(c, R.Image(tables["rnodes"], tables["rkids"]))
    filters = R.edit_filters(c)

    def rstats():
        s = eng.debug_tables()["rstats"]
        return int(s[0]), int(s[1])

    for label, op, arg, how in R.edit_script(proof["clear"][0]):
        before = rstats()
        if op == "set":
            eng.retain_set(*arg)
            rt.insert(*arg)
        elif op == "remove":
            assert eng.retain_remove(arg) == rt.remove(arg)
        elif op == "remove_batch":
            want_old = [None if orc.topic_parse(t) is None else rt.remove(t) for t in arg]
            old, n_removed = eng.retain_remove_batch(*R.pack(arg))
            assert n_removed == R.REMOVE_BATCH_REMOVED == sum(x is not None for x in want_old)
            assert old.tolist() == [R.VMAX if x is None else x for x in want_old]
            assert old[0] == old[2] == R.VMAX and want_old[0] == R.VMAX and want_old[2] is None   # indistinguishable in old_values
        else:
            eng.compact()
        _check(eng, rt, filters, label)
        after = rstats()
        if how == "patch":
            assert after[0] == before[0] and after[1] > before[1], (label, before, after)
        elif how == "flatten":
            assert after[0] == before[0] + 1, (label, before, after)
    _check(eng, rt, c.filters() + ["#", "+/#", "$c/#"], "all filters after the edits")
    eng.debug_knob("retain_caps", R.RQ)
    _check(eng, rt, filters + c.filters(heavy=False), "from 64 entries after the edits")
    eng.close()
