"""CPU tier: the small-graph form of the retained lookup (engine.cu small_graph_retain) on the emulated kernels.  The launch is
sized for a CAPACITY and the real filter count and text length come from a header in memory: k_retain_init must stop at
the real count, k_retain_scan must scan only the real count, and launch_retain must hand the header to the tokeniser.
Rows past the batch are poisoned (garbage offsets, a status / span pattern that must survive, a stale valid `#` in their
token rows), so a launch that touches them fails.  The tests/_retain_edges.py corpus runs at capacity n + 37 and at both
tier capacities (64 and 2048 filters); lists and per-round task counts must equal the pipelined form's.  The driver is
tests/native/emu/emu_retain_graph.cpp: the emulator driver plus the graph-form export."""
import ctypes as C
import shutil
import subprocess
import sys

import numpy as np
import pytest

import _retain_edges as R
from oracle import oracle as orc
from rmqtt_b200.engine import MatchResult, pack
from test_emu_kernels import CSRC, EMU, ROOT, Emu, _emu_retained_load, _same

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

TIERS = (64, 2048)            # engine.cu small_graph_tier: filters per tier


def _build(tmp, san: bool):
    """tests/native/emu/emu_retain_graph.cpp with the real kernel sources on the CPU emulation, built like test_emu_kernels._build"""
    out = tmp / ("libemu_rgraph_asan.so" if san else "libemu_rgraph.so")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-DGM_CPU_EMU", f"-I{EMU}", f"-I{CSRC}", "-shared", "-fPIC", "-pthread", "-fno-omit-frame-pointer",
           *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"] if san else []),
           "-o", str(out), str(EMU / "emu_retain_graph.cpp"), str(CSRC / "host_trie.cpp"), str(CSRC / "retain_tree.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr and "cannot find" in r.stderr:
        pytest.skip("sanitizer runtime not installed")
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _lib(path):
    lib = C.CDLL(str(path))
    lib.emu_new.restype = C.c_void_p
    for f in ("emu_retain_set", "emu_retain_match", "emu_retain_match_graph"):
        getattr(lib, f).restype = C.c_int32
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _lib(_build(tmp_path_factory.mktemp("emu_rg"), san=False))


def _lookup(e, filters, rows=None, caps=1 << 14):
    """-> (MatchResult, tasks per round, descriptors) through emu_retain_match (rows None) or its graph form at `rows`;
    the scratch grows on overflow as gm_engine::run_retain grows it"""
    fb, fo = pack(filters)
    n = len(fo) - 1
    spans, status = np.zeros((n, 2), dtype=np.uint32), np.zeros(n, dtype=np.int32)
    work, needed = np.zeros(2, dtype=np.uint64), C.c_uint64(0)
    fb = np.ascontiguousarray(fb if len(fb) else np.zeros(1, np.uint8))
    cap, items, descs = 1024, caps, caps
    for _ in range(40):
        ids = np.zeros(cap, dtype=np.uint32)
        args = [e.h, C.c_void_p(fb.ctypes.data), C.c_void_p(fo.ctypes.data), C.c_uint64(n)]
        tail = [0, items, descs, C.c_void_p(spans.ctypes.data), C.c_void_p(ids.ctypes.data), C.c_uint64(cap), C.byref(needed),
                C.c_void_p(status.ctypes.data), C.c_void_p(work.ctypes.data)]
        rc = e.lib.emu_retain_match(*args, *tail) if rows is None else e.lib.emu_retain_match_graph(*args, rows, *tail)
        if rc == -3:
            cap = int(needed.value) + 16
        elif rc <= -100:
            items *= 4 if (-rc - 100) & 1 else 1
            descs *= 4 if (-rc - 100) & 2 else 1
        else:
            assert rc == 0, (rows, rc)
            tasks, nd = e.retain_tasks()
            return MatchResult(spans, ids[:int(needed.value)], status, int(needed.value)), tasks, nd
    raise AssertionError("no convergence")


def _graph_equals_pipelined(e, rt, filters, what, caps=1 << 14):
    want = rt.match_batch(*pack(filters))
    res0, tasks0, nd0 = _lookup(e, filters, caps=caps)
    _same(res0, want)
    n = len(filters)
    for rows in [n + 37] + [t for t in TIERS if t >= n]:
        res, tasks, nd = _lookup(e, filters, rows, caps=caps)
        try:
            _same(res, want)
            assert (res.status == res0.status).all()
            assert (res.spans[:, 1] == res0.spans[:, 1]).all() and res.needed == res0.needed
            assert tasks == tasks0 and nd == nd0, (tasks, tasks0, nd, nd0)
        except AssertionError as ex:
            raise AssertionError(f"{what} at {rows} rows: {ex}") from None


def _corpus_run(lib, how, light=False):
    R.check_constants()
    for c in (R.retained_edge_corpus(), R.retained_lit_hash_corpus()):
        e, rt = Emu(lib), c.load_oracle(orc)
        _emu_retained_load(lib, e, c, how)
        _graph_equals_pipelined(e, rt, c.filters(heavy=not light), f"{how}: all filters")
        for q in c.stated():
            if q.heavy and light:
                continue
            _graph_equals_pipelined(e, rt, [q.filt], f"{how}: {q.filt}")
        if c.bulk and not light:
            for n in (1, 64, 65, 2048):
                _graph_equals_pipelined(e, rt, c.batch(n), f"{how}: batch of {n}")
        _graph_equals_pipelined(e, rt, c.filters(heavy=False)[:60], f"{how}: from 64 entries", caps=R.RQ)
        e.close()


@pytest.mark.parametrize("how", ["set", "bulk"])
def test_graph_form_equals_pipelined_form_on_the_retained_corpus(emu, how):
    _corpus_run(emu, how)


def test_rows_past_the_batch_stay_untouched_and_the_capacity_is_checked(emu):
    """A stale valid `#` row right behind a one-filter batch, the smallest capacity (= n), and rows < n refused."""
    c = R.retained_edge_corpus()
    e, rt = Emu(emu), c.load_oracle(orc)
    _emu_retained_load(emu, e, c, "bulk")
    for filters in (["w/k9/+"], ["#"], ["a+"], [""], ["pi/+", "$c/#", "nope"]):
        want = rt.match_batch(*pack(filters))
        for rows in (len(filters), len(filters) + 1, 64):
            res, _, _ = _lookup(e, filters, rows)
            _same(res, want)
    fb, fo = pack(["a", "b"])
    spans, status, ids, needed = np.zeros((2, 2), np.uint32), np.zeros(2, np.int32), np.zeros(4, np.uint32), C.c_uint64(0)
    rc = emu.emu_retain_match_graph(e.h, C.c_void_p(fb.ctypes.data), C.c_void_p(fo.ctypes.data), C.c_uint64(2), 1, 0, 1 << 14, 1 << 14,
                                    C.c_void_p(spans.ctypes.data), C.c_void_p(ids.ctypes.data), C.c_uint64(4), C.byref(needed),
                                    C.c_void_p(status.ctypes.data), None)
    assert rc == -2
    e.close()


def test_graph_form_under_asan_ubsan(tmp_path):
    """The graph form compiled with AddressSanitizer + UBSan, in a subprocess (the sanitizer runtime must be loaded first):
    the light corpus, bulk-loaded, at n + 37 and both tier capacities."""
    so = _build(tmp_path, san=True)
    script = tmp_path / "run.py"
    script.write_text(f"""
import sys
sys.path.insert(0, {str(ROOT)!r}); sys.path.insert(0, {str(ROOT / 'tests')!r})
import test_emu_retain_graph as T
T._corpus_run(T._lib({str(so)!r}), "bulk", light=True)
print("asan run ok")
""")
    libasan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    env = {"PATH": "/usr/bin:/bin", "LD_PRELOAD": libasan, "ASAN_OPTIONS": "detect_leaks=0:detect_stack_use_after_return=0", "PYTHONPATH": str(ROOT)}
    import os
    for k in ("HOME", "LD_LIBRARY_PATH", "VIRTUAL_ENV"):
        if k in os.environ:
            env[k] = os.environ[k]
    run = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=1500, env=env)
    assert run.returncode == 0 and "asan run ok" in run.stdout, (run.stdout[-1500:], run.stderr[-4000:])
