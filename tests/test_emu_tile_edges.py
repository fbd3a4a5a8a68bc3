"""CPU tier of the fast path's id expansion (k_match_fast's publish -> k_match_expand) at its tile and capacity edges: the
corpus of tests/_tile_edges.py through the emulated kernels, into GUARDED output buffers — [guard | cap | guard] filled with a
position-dependent pattern — on POISONED scratch (the driver clears only what the engine clears), on a scratch KEPT across
calls as a match context keeps it, in the small-graph form and in the pipelined host call's chunks.

After every call: both guards of the ids, spans and status are intact; a successful ids-mode call's spans of the OK rows are
pairwise disjoint and tile [0, needed) exactly, no pattern word is left inside it, and every row's multiset equals the oracle;
a call with cap < needed returns the capacity error with the exact `needed` and writes nothing at or past cap."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import _tile_edges as T
from rmqtt_b200.engine import MatchResult
from test_emu_kernels import ROOT, Emu, _build, _emu_load_corpus

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

ERR_CAPACITY, ERR_SCRATCH = -3, -60
F_DESC, F_BULK, F_STATS, F_GRAPH, F_RAW = 1, 2, 4, 16, 32
MP_DIAG_NO_PUBLISH = 2


def _setup(lib):
    lib.emu_new.restype = C.c_void_p
    lib.emu_bulk_load.restype = C.c_uint64
    for f in ("emu_sub_add", "emu_match_ex", "emu_match_chunked"):
        getattr(lib, f).restype = C.c_int32
    return lib


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return _setup(C.CDLL(str(_build(tmp_path_factory.mktemp("emu_tiles"), san=False))))


class Guarded:
    """[guard | n | guard] elements of `width` u32 words, filled with the position pattern."""

    def __init__(self, n, width=1, guard=64, salt=0):
        self.n, self.w, self.g = n, width, guard
        self.fill = T.pattern((n + 2 * guard) * width, salt)
        self.buf = self.fill.copy()
        self.inner = self.buf[guard * width:(guard + n) * width]
        self.ptr = C.c_void_p(self.inner.ctypes.data)

    def guards_intact(self):
        g = self.g * self.w
        return bool((self.buf[:g] == self.fill[:g]).all() and (self.buf[len(self.buf) - g:] == self.fill[len(self.buf) - g:]).all())

    def pristine(self, lo=0, hi=None):
        """elements [lo, hi) of the inner range still hold the pattern"""
        hi = self.n if hi is None else hi
        return bool((self.inner[lo * self.w:hi * self.w] == self.fill[(self.g + lo) * self.w:(self.g + hi) * self.w]).all())

    def written(self, lo, hi):
        """no element of [lo, hi) still holds its pattern word"""
        a = self.inner[lo * self.w:hi * self.w].reshape(-1, self.w)
        b = self.fill[(self.g + lo) * self.w:(self.g + hi) * self.w].reshape(-1, self.w)
        return not bool((a == b).all(axis=1).any())


class Ctx:
    def __init__(self, lib):
        self.lib = lib
        self.c = T.tile_corpus()
        self.tree = self.c.load_oracle()
        T.check_against_oracle(self.c, self.tree)
        self.e = Emu(lib)
        lib.emu_set_pool_rows(self.e.h, T.K2_POOL_ROWS)
        _emu_load_corpus(lib, self.e, self.c)
        self.want = {}
        self.exact = False           # no guards: buffers of exactly the offered size (the ASan run: it sees their ends)

    def batch(self, name):
        if name not in self.want:
            tb, to = self.c.packed(name)
            w = self.tree.match_batch(tb, to)
            ids = w["ids"].copy()
            for i in range(len(w["offsets"]) - 1):
                ids[w["offsets"][i]:w["offsets"][i + 1]].sort()
            self.want[name] = (tb, to, w["counts"], ids, w["counters"])
        return self.want[name]

    def knobs(self, tile_chunk=1, k2_ctas=0, diag=0, graph_cap=0):
        self.lib.emu_set_knobs(self.e.h, tile_chunk, k2_ctas, diag, graph_cap)

    def call(self, name, flags, cap, guard=None, chunk=0):
        """One call into guarded buffers -> (rc, needed, ids, spans, status, work, deferred)"""
        tb, to, counts, _, _ = self.batch(name)
        n = len(to) - 1
        guard = 0 if self.exact else guard if guard is not None else max(64, int(counts.clip(0).sum()) + 64)
        width = 2 if flags & F_DESC and flags & F_RAW else 1
        g = 0 if self.exact else 64
        ids, spans, status = Guarded(cap, width, guard, 1), Guarded(n, 2, g, 2), Guarded(n, 1, g, 3)
        needed, deferred = C.c_uint64(0), C.c_uint32(0)
        work = np.zeros(4, dtype=np.uint64)
        blob = np.ascontiguousarray(tb if len(tb) else np.zeros(1, np.uint8))
        if chunk:
            rc = self.lib.emu_match_chunked(self.e.h, C.c_void_p(blob.ctypes.data), C.c_void_p(to.ctypes.data), C.c_uint64(n), flags, C.c_uint64(chunk), spans.ptr, ids.ptr,
                                            C.c_uint64(cap), C.byref(needed), status.ptr)
        else:
            rc = self.lib.emu_match_ex(self.e.h, C.c_void_p(blob.ctypes.data), C.c_void_p(to.ctypes.data), C.c_uint64(n), None, C.c_uint64(n), None, flags, spans.ptr, ids.ptr,
                                       C.c_uint64(cap), C.byref(needed), status.ptr, C.c_void_p(work.ctypes.data), C.byref(deferred))
        return rc, int(needed.value), ids, spans, status, work, int(deferred.value)


@pytest.fixture(scope="module")
def ctx(lib):
    x = Ctx(lib)
    yield x
    x.e.close()


def _total(x, name, desc=False):
    return sum(c.F or 0 for c in x.c.batches[name]) if desc else int(x.batch(name)[2].clip(0).sum())


def check_exact(x, name, r, what):
    """A successful ids-mode call: guards, status, the spans tile [0, needed) exactly, no pattern left, per-row multisets."""
    rc, needed, ids, spans, status, _, _ = r
    _, _, counts, wids, _ = x.batch(name)
    total = int(counts.clip(0).sum())
    assert rc == 0 and needed == total, (what, rc, needed, total)
    assert ids.guards_intact() and spans.guards_intact() and status.guards_intact(), f"{what}: a guard was written"
    st = status.inner.view(np.int32)
    assert (st == np.where(counts < 0, -2, 0)).all(), f"{what}: status"
    sp = spans.inner.reshape(-1, 2)
    ok = (st == 0) & (sp[:, 1] > 0)
    assert (sp[st == 0, 1] == counts[st == 0]).all(), f"{what}: span lengths"
    off, cnt = sp[ok, 0].astype(np.int64), sp[ok, 1].astype(np.int64)
    o = np.argsort(off, kind="stable")
    ends = np.cumsum(cnt[o])
    assert (off[o] == ends - cnt[o]).all() and (ends[-1] if len(ends) else 0) == needed, f"{what}: the spans do not tile [0, needed)"
    assert ids.written(0, needed), f"{what}: a pattern word is left inside [0, needed)"
    got_c, got_i = MatchResult(sp, ids.inner, st, needed).canonical()
    assert (got_c == counts).all() and len(got_i) == len(wids) and (got_i == wids).all(), f"{what}: id multisets differ"


def check_capacity(x, name, r, cap, what, desc=False):
    rc, needed, ids, spans, status, _, _ = r
    assert rc == ERR_CAPACITY and needed == _total(x, name, desc), (what, cap, rc, needed)
    assert ids.guards_intact() and spans.guards_intact() and status.guards_intact(), f"{what}: cap {cap}: written at or past cap"


def caps_below(x, name):
    """needed - 1, needed - the last tile's ids (rows in the emulator's order), needed / 2 and / 3 (some tiles fit, others
    do not), 0"""
    total = _total(x, name)
    last = [t for t in x.c.tile_ids(name) or [] if t][-1:] or [0]     # (order not known: that cap is left out)
    return sorted({c for c in (total - 1, total - last[0], total // 2, total // 3, 0) if 0 <= c < total}, reverse=True)


def run_shapes(x, names=T.SHAPES, flags=(0, F_BULK, F_STATS)):
    for name in names:
        total = _total(x, name)
        for fl in flags:
            r = x.call(name, fl, total)
            check_exact(x, name, r, f"{name} flags {fl}")
            assert r[6] == x.c.n_deferred(name), (name, r[6])
            if fl & F_STATS:
                k = x.batch(name)[4]
                assert [int(v) for v in r[5]] == [k["V"], k["E"], k["F"], k["M"]], name
        for cap in caps_below(x, name):
            check_capacity(x, name, x.call(name, 0, cap), cap, name)


def run_descriptors(x, names):
    """Descriptor mode: the raw descriptors into a guarded buffer (geometry, F and the ids per row they stand for), then
    expanded to ids; and its capacity edges."""
    for name in names:
        cases = x.c.batches[name]
        nd = _total(x, name, desc=True)
        rc, needed, descs, spans, status, _, _ = r = x.call(name, F_DESC | F_RAW, nd)
        assert rc == 0 and needed == nd and descs.guards_intact() and spans.guards_intact() and status.guards_intact(), (name, rc, needed, nd)
        sp = spans.inner.reshape(-1, 2)
        d = descs.inner.reshape(-1, 2)
        assert descs.written(0, needed), f"{name}: a pattern pair is left among the descriptors"
        valid = np.asarray([c.F is not None for c in cases])
        assert (sp[valid, 1] == [c.F for c in cases if c.F is not None]).all(), name
        used = valid & (sp[:, 1] > 0)                   # (an empty span's offset is arbitrary)
        o = np.argsort(sp[used, 0], kind="stable")
        ends = np.cumsum(sp[used, 1][o].astype(np.int64))
        assert (sp[used, 0][o] == ends - sp[used, 1][o]).all() and (ends[-1] if len(ends) else 0) == needed, name
        for i, c in enumerate(cases):
            if c.F:
                assert int(d[sp[i, 0]:sp[i, 0] + sp[i, 1], 1].astype(np.int64).sum()) == c.M, (name, c.topic)
        check_exact(x, name, x.call(name, F_DESC, _total(x, name)), f"{name} descriptors expanded")
        for cap in sorted({nd - 1, nd // 2, 0} - {nd}):
            if cap >= 0:
                check_capacity(x, name, x.call(name, F_DESC | F_RAW, cap), cap, f"{name} descriptors", desc=True)


def check_no_publish(x, name, r, what):
    """diag_flags = MP_DIAG_NO_PUBLISH: the fast path writes no id (only the deferred topics' spans hold ids, exact ones),
    `needed` and the span lengths are still exact."""
    rc, needed, ids, spans, status, _, _ = r
    _, _, counts, wids, _ = x.batch(name)
    assert rc == 0 and needed == _total(x, name) and ids.guards_intact() and spans.guards_intact() and status.guards_intact(), (what, rc, needed)
    sp, st = spans.inner.reshape(-1, 2), status.inner.view(np.int32)
    assert (sp[st == 0, 1] == counts[st == 0]).all(), what
    written = np.zeros(ids.n, dtype=bool)
    wo = np.concatenate([[0], np.cumsum(counts.clip(0))])
    for i, c in enumerate(x.c.batches[name]):
        if c.deferred:
            written[sp[i, 0]:sp[i, 0] + sp[i, 1]] = True
            assert (np.sort(ids.inner[sp[i, 0]:sp[i, 0] + sp[i, 1]]) == wids[wo[i]:wo[i + 1]]).all(), (what, c.topic)
    assert (ids.inner[~written] == ids.fill[ids.g:ids.g + ids.n][~written]).all(), f"{what}: the fast path wrote ids"


def run_no_publish(x, names):
    """MP_DIAG_NO_PUBLISH, then without it: exact again."""
    for name in names:
        x.knobs(diag=MP_DIAG_NO_PUBLISH)
        try:
            r = x.call(name, 0, _total(x, name))
        finally:
            x.knobs()
        check_no_publish(x, name, r, name)
        check_exact(x, name, x.call(name, 0, _total(x, name)), f"{name} after no-publish")


def run_kept_graph(x):
    """One scratch kept across calls: a poison batch of a tier's capacity in rows fills the tile records and items, then the
    small batches run in the small-graph form (launched for that capacity) on them."""
    x.lib.emu_keep_scratch(x.e.h, 1)
    try:
        for cap_n, poison, small in ((64, "z64", ("g0_low", "g0_at", "p1", "p33", "p63")), (2048, "z2048", ("g1_low", "g1_at", "p65", "items1024"))):
            for name in small:
                for fl in (0, F_STATS):
                    x.knobs()
                    check_exact(x, poison, x.call(poison, 0, _total(x, poison)), poison)
                    x.knobs(graph_cap=cap_n)
                    g = _total(x, poison) + 64
                    r = x.call(name, F_GRAPH | fl, _total(x, name), guard=g)
                    check_exact(x, name, r, f"{name} graph form at {cap_n} on kept scratch")
                    if fl & F_STATS:
                        k = x.batch(name)[4]
                        assert [int(v) for v in r[5]] == [k["V"], k["E"], k["F"], k["M"]], name
                x.knobs(graph_cap=cap_n)
                for cap in caps_below(x, name):
                    check_capacity(x, name, x.call(name, F_GRAPH, cap, guard=_total(x, poison) + 64), cap, f"{name} graph form")
    finally:
        x.knobs()
        x.lib.emu_keep_scratch(x.e.h, 0)


def run_chunked(x):
    """The pipelined host call: chunks share the bump cursor over the ids, every chunk has its own item array."""
    for name, chunk in (("full32", 32), ("full32", 64), ("p2049", 1024), ("holes", 64), ("singles", 32)):
        total = _total(x, name)
        check_exact(x, name, x.call(name, 0, total, chunk=chunk), f"{name} in chunks of {chunk}")
        for cap in caps_below(x, name):
            check_capacity(x, name, x.call(name, 0, cap, chunk=chunk), cap, f"{name} in chunks of {chunk}")


def test_tile_corpus_reaches_its_shapes(ctx):
    """(the Ctx checks the corpus against the oracle: F, M, validity, the value sets per tile)"""
    assert ctx.c.n_deferred("holes") == 9 and ctx.c.tiles("items1024") == [1024]


def test_tile_shapes_exact_guarded_and_at_capacity(ctx):
    run_shapes(ctx)


def test_scheduling_knobs(ctx):
    for tc, k2 in ((7, 0), (1024, 0), (1, 1), (1, 3), (7, 1)):
        ctx.knobs(tile_chunk=tc, k2_ctas=k2)
        try:
            run_shapes(ctx, ("holes", "full32", "p2049", "singles"), flags=(0,))
        finally:
            ctx.knobs()


def test_descriptor_mode_guarded(ctx):
    run_descriptors(ctx, ("items1024", "full32", "step_big", "singles", "holes", "p65", "p2049"))


def test_no_publish_diagnostic(ctx):
    run_no_publish(ctx, ("items65", "holes", "full32", "p2049"))


def test_small_graph_form_on_a_kept_scratch(ctx):
    run_kept_graph(ctx)


def test_pipelined_chunks_on_one_kept_scratch(ctx):
    run_chunked(ctx)


def test_tile_edges_under_asan_ubsan(tmp_path):
    """The same checks in the AddressSanitizer + UBSan build, with exactly sized output buffers (the guards catch what lands
    next to them, ASan what lands beyond)."""
    so = _build(tmp_path, san=True)
    script = tmp_path / "run.py"
    script.write_text(f"""
import sys, ctypes as C
sys.path.insert(0, {str(ROOT)!r}); sys.path.insert(0, {str(ROOT / 'tests')!r})
import test_emu_tile_edges as X
x = X.Ctx(X._setup(C.CDLL({str(so)!r})))
x.exact = True
X.run_shapes(x, ("items1024", "full32", "step_big", "singles", "holes", "p33", "p2049", "g1_at"), flags=(0,))
X.run_descriptors(x, ("full32", "holes"))
X.run_no_publish(x, ("full32",))
X.run_kept_graph(x)
X.run_chunked(x)
x.e.close()
print("asan run ok")
""")
    libasan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    env = {"PATH": "/usr/bin:/bin", "LD_PRELOAD": libasan, "ASAN_OPTIONS": "detect_leaks=0:detect_stack_use_after_return=0", "PYTHONPATH": str(ROOT)}
    for k in ("HOME", "LD_LIBRARY_PATH", "VIRTUAL_ENV"):
        if k in os.environ:
            env[k] = os.environ[k]
    run = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=1500, env=env)
    assert run.returncode == 0 and "asan run ok" in run.stdout, (run.stdout[-1500:], run.stderr[-4000:])
