"""CPU tier: expiry of retained messages (gm_retain_set_ttl, gm_retain_bulk_load_ttl, gm_retain_remove_expired,
gm_retain_match_batch_at).

* The bookkeeping on a GM_FLAG_HOST_ONLY engine against tests/_retain_expiry.py's restatement of the reference: which handles
  the sweep returns (cap 0, 1, exactly the expired count), the duplicate-handle error, re-sets, removals, gm_compact in between.
* The lookup on the emulated kernels (tests/native/emu/emu_retain_expiry.cpp), pipelined and in the small-graph form, and
  again under ASan + UBSan: bit-exact against get_message(now) over the retained boundary corpus with seeded deadlines (none,
  past, exactly now, future), `#` ranges fully, partly and not at all expired, `$` roots, literal-`#` shadowing (mode-2 tasks),
  filters deeper than 8 levels, and rows past the batch left untouched."""
import ctypes as C
import random
import shutil
import subprocess

import numpy as np
import pytest

import _retain_edges as R
from _retain_expiry import TimedRetain, seeded_deadlines
from oracle import oracle as orc
from rmqtt_b200 import _native as N
from rmqtt_b200.engine import Engine, GpuMqttError, MatchResult, pack
from test_emu_kernels import CSRC, EMU, ROOT, _Env, _canon

NOW = 1_760_000_000_000          # ms since the Unix epoch


# ---- bookkeeping on a host-only engine -------------------------------------------------------------------------------
def _sweep_all(eng, now, cap=1 << 20):
    return sorted(eng.retain_remove_expired(now, cap).tolist())


def test_sweep_returns_the_expired_handles_earliest_first_with_cap_edges():
    eng = Engine(host_only=True)
    deadlines = {10 + i: NOW - 50 + 10 * i for i in range(10)}          # 5 past, NOW exactly (i = 5), 4 future
    for h, d in deadlines.items():
        eng.retain_set(f"s/{h}", h, deadline_ms=d)
    eng.retain_set("s/plain", 99)
    expired = sorted(h for h, d in deadlines.items() if NOW >= d)
    assert len(expired) == 6
    assert eng.retain_remove_expired(NOW, 0).tolist() == []
    assert eng.retain_remove_expired(NOW, 1).tolist() == [10]           # the earliest deadline
    assert sorted(eng.retain_remove_expired(NOW, 5).tolist()) == expired[1:]   # exactly the remaining expired count
    assert eng.retain_remove_expired(NOW, 5).tolist() == []
    assert eng.stats()["retained_values"] == 1 + 4
    assert _sweep_all(eng, NOW + 10_000) == [16, 17, 18, 19]
    assert eng.stats()["retained_values"] == 1


def test_a_handle_with_a_deadline_lives_under_one_topic():
    eng = Engine(host_only=True)
    eng.retain_set("a/1", 5, deadline_ms=NOW)
    for call in (lambda: eng.retain_set("a/2", 5), lambda: eng.retain_set("a/2", 5, deadline_ms=NOW + 1)):
        with pytest.raises(GpuMqttError) as ei:
            call()
        assert ei.value.code == N.GM_ERR_INVALID_ARG
    assert eng.stats()["retained_values"] == 1                           # nothing changed
    blob, offs = pack(["b/1", "a/2"])
    with pytest.raises(GpuMqttError) as ei:
        eng.retain_bulk_load(blob, offs, np.array([7, 5], np.uint32), np.array([0, 0], np.uint64))
    assert ei.value.code == N.GM_ERR_INVALID_ARG
    blob, offs = pack(["b/1", "b/2"])
    with pytest.raises(GpuMqttError):                                    # the same handle twice with a deadline in one batch
        eng.retain_bulk_load(blob, offs, np.array([8, 8], np.uint32), np.array([NOW, NOW], np.uint64))
    with pytest.raises(GpuMqttError):
        eng.retain_set("c", 1 << 28, deadline_ms=NOW)                   # GM_RETAIN_TTL_MAX_HANDLE
    assert eng.stats()["retained_values"] == 1
    assert _sweep_all(eng, NOW) == [5]
    eng.retain_set("a/2", 5)                                             # once removed, the handle is free again


def test_reset_clears_or_replaces_and_removal_clears():
    eng = Engine(host_only=True)
    eng.retain_set("a", 1, deadline_ms=NOW)
    eng.retain_set("a", 1)                                               # set_with_timeout(.., None): no deadline any more
    eng.retain_set("b", 2, deadline_ms=NOW)
    eng.retain_set("b", 2, deadline_ms=NOW + 100)                        # replaced
    eng.retain_set("c", 3, deadline_ms=NOW)
    assert eng.retain_remove("c") == 3                                   # removal clears it ...
    eng.retain_set("c2", 3)                                              # ... so the handle may live elsewhere, without one
    eng.retain_set("d", 4, deadline_ms=NOW)
    eng.retain_set("d", 5)                                               # replaced by another handle: 4 loses its deadline
    eng.retain_set("d2", 4)
    assert _sweep_all(eng, NOW) == []
    assert _sweep_all(eng, NOW + 100) == [2]
    assert eng.stats()["retained_values"] == 4                           # a, c2, d, d2


def test_bulk_load_ttl_equals_set_ttl_calls_in_order_on_both_builds():
    rng = random.Random(3)
    rows = []
    for i in range(3000):
        t = f"r/{rng.randrange(40)}/{rng.randrange(60)}"
        rows.append((t, rng.randrange(1, 5000), rng.choice([0, 0, NOW - 5, NOW, NOW + 5])))
    for parallel in (True, False):
        eng, ref = Engine(host_only=True), TimedRetain(orc)
        if not parallel:
            eng.retain_set("seed", 0)
            ref.set_with_timeout("seed", 0)
        # keep the batch valid: a handle with a deadline appears under one topic only
        used, ok = {}, []
        for t, h, d in rows:
            if used.get(h, t) != t:
                continue
            used[h] = t
            ok.append((t, h, d))
        blob, offs = pack([t for t, _, _ in ok])
        with _Env(GM_HOST_PAR_MIN=1, GM_HOST_THREADS=4):
            n = eng.retain_bulk_load(blob, offs, np.array([h for _, h, _ in ok], np.uint32), np.array([d for _, _, d in ok], np.uint64))
        assert n == len(ok)
        for t, h, d in ok:
            ref.set_with_timeout(t, h, d)
        assert eng.stats()["retained_values"] == ref.rt.values_size()
        assert _sweep_all(eng, NOW - 1) == ref.remove_expired_messages(NOW - 1)
        assert _sweep_all(eng, NOW) == ref.remove_expired_messages(NOW)
        assert _sweep_all(eng, NOW + 10) == ref.remove_expired_messages(NOW + 10)
        assert eng.stats()["retained_values"] == ref.rt.values_size()


def test_seeded_rounds_with_compaction_against_the_reference():
    rng = random.Random(11)
    eng, ref = Engine(host_only=True), TimedRetain(orc)
    eng.add("x/+", 1)
    now = NOW
    for rnd in range(30):
        for _ in range(200):
            t = f"m/{rng.randrange(30)}/{rng.randrange(30)}"
            op = rng.random()
            if op < 0.45:
                h = rng.randrange(1, 4000)
                d = rng.choice([0, now + rng.randrange(-50, 200)])
                owner = next((tt for tt, hh in ref.val.items() if hh == h), None)
                if owner is not None and owner != t:
                    if h in ref.dl:                              # a handle with a deadline stays under its topic
                        with pytest.raises(GpuMqttError):
                            eng.retain_set(t, h, deadline_ms=d)
                    continue                                     # (every handle stays under one topic here)
                eng.retain_set(t, h, deadline_ms=d)
                ref.set_with_timeout(t, h, d)
            elif op < 0.7:
                assert eng.retain_remove(t) == ref.remove(t)
            else:
                cap = rng.choice([0, 1, 3, 1 << 20])
                got = eng.retain_remove_expired(now, cap).tolist()
                want = ref.expired_handles(now)
                assert len(got) == min(cap, len(want)) and set(got) <= set(want)
                for h in got:
                    ref.remove(next(tt for tt, hh in ref.val.items() if hh == h))
        if rnd % 7 == 3:
            eng.compact()
        now += 37
        assert eng.stats()["retained_values"] == ref.rt.values_size()
    assert _sweep_all(eng, now + 1000) == ref.remove_expired_messages(now + 1000)


def test_republishing_the_same_handle_without_a_deadline_leaves_the_device_copy_clean():
    eng = Engine(host_only=True)
    eng.retain_set("a/b", 7)
    eng.retain_set("a/c", 8, deadline_ms=NOW)                            # the engine holds deadlines
    eng.flush()
    p0 = eng.stats()["pending"]
    eng.retain_set("a/b", 7)                                             # same topic, same handle, no deadline before or after
    assert eng.stats()["pending"] == p0
    eng.retain_set("a/c", 8, deadline_ms=NOW)                            # the same deadline again
    assert eng.stats()["pending"] == p0
    eng.retain_set("a/c", 8, deadline_ms=NOW + 1)
    assert eng.stats()["pending"] == 1


# ---- the lookup on the emulated kernels --------------------------------------------------------------------------------
def _lib(path):
    lib = C.CDLL(str(path))
    lib.emu_new.restype = C.c_void_p
    for f in ("emu_retain_set_ttl", "emu_retain_set", "emu_retain_match_at"):
        getattr(lib, f).restype = C.c_int32
    for f in ("emu_retain_bulk_load_ttl", "emu_retain_remove_expired"):
        getattr(lib, f).restype = C.c_uint64
    return lib


def _build(tmp, san):
    out = tmp / ("libemu_rexp_asan.so" if san else "libemu_rexp.so")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-DGM_CPU_EMU", f"-I{EMU}", f"-I{CSRC}", "-shared", "-fPIC", "-pthread", "-fno-omit-frame-pointer",
           *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"] if san else []),
           "-o", str(out), str(EMU / "emu_retain_expiry.cpp"), str(CSRC / "host_trie.cpp"), str(CSRC / "retain_tree.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr and "cannot find" in r.stderr:
        pytest.skip("sanitizer runtime not installed")
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def rexp(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    return _lib(_build(tmp_path_factory.mktemp("rexp"), san=False))


class _E:
    def __init__(self, lib):
        self.lib, self.h = lib, C.c_void_p(lib.emu_new())

    def close(self):
        self.lib.emu_free(self.h)

    def set(self, t, v, d=0):
        b = t.encode()
        assert self.lib.emu_retain_set_ttl(self.h, b, len(b), v, C.c_uint64(d)) == 0, t

    def match(self, filters, now, rows=0, cap=None, caps=1 << 14):
        """-> (rc, MatchResult, needed); the scratch grows on overflow as gm_engine::run_retain grows it"""
        blob, offs = pack(filters)
        n = len(offs) - 1
        blob = np.ascontiguousarray(blob if len(blob) else np.zeros(1, np.uint8))
        spans, status, needed = np.zeros((n, 2), np.uint32), np.zeros(n, np.int32), C.c_uint64(0)
        items = descs = caps
        c = 1 << 16 if cap is None else cap
        while True:
            ids = np.full(c + 64, 0xEEEEEEEE, dtype=np.uint32)          # poisoned beyond the output
            rc = self.lib.emu_retain_match_at(self.h, C.c_uint64(now), C.c_void_p(blob.ctypes.data), C.c_void_p(offs.ctypes.data), C.c_uint64(n), rows, items, descs,
                                              C.c_void_p(spans.ctypes.data), C.c_void_p(ids.ctypes.data), C.c_uint64(c), C.byref(needed), C.c_void_p(status.ctypes.data))
            if rc <= -100:
                err = -rc - 100
                items *= 4 if err & 1 else 1
                descs *= 4 if err & 2 else 1
                continue
            if rc == -3 and cap is None:
                c = int(needed.value) + 16
                continue
            return rc, MatchResult(spans, ids[:int(needed.value)], status, int(needed.value)), ids, int(needed.value)


def _same(res, want, what):
    counts, ids = res.canonical()
    wc, wi = _canon(want)
    assert (counts == wc).all(), f"{what}: counts differ at {np.nonzero(counts != wc)[0][:5]}"
    assert len(ids) == len(wi) and (ids == wi).all(), what


def _ttl_cases(ref, e, rng, now):
    """`#` ranges fully, partly and not at all expired, below and at the root, deeper than 8 levels"""
    deep = "/".join(f"d{i}" for i in range(11))
    base = 1 << 20
    for i in range(40):
        for t, d in ((f"xf/{i}", now - 1 - i), (f"xn/{i}", 0), (f"xp/{i}", (now, now + 5, 0, now - 3)[i % 4]), (f"{deep}/{i}", (now, 0)[i % 2])):
            h = base
            base += 1
            e.set(t, h, d)
            ref.set_with_timeout(t, h, d)
    return ["xf/#", "xn/#", "xp/#", "xp/+", "+/#", "#", "+/+", f"{deep}/#", f"{deep}/+", "/".join(["+"] * 11) + "/#", deep + "/7"]


def _load(lib, c, how, now, rng):
    e, ref = _E(lib), TimedRetain(orc)
    dls = seeded_deadlines(c.all_topics(), now, rng)
    rows = c.all_topics()
    if how == "set":
        for t, v in rows:
            e.set(t, v, dls.get(v, 0))
    else:
        blob, offs = pack([t for t, _ in rows])
        vals = np.array([v for _, v in rows], np.uint32)
        dl = np.array([dls.get(v, 0) for _, v in rows], np.uint64)
        with _Env(GM_HOST_PAR_MIN=1, GM_HOST_THREADS=4):
            assert lib.emu_retain_bulk_load_ttl(e.h, C.c_void_p(blob.ctypes.data), C.c_void_p(offs.ctypes.data), C.c_void_p(vals.ctypes.data),
                                                C.c_void_p(dl.ctypes.data), C.c_uint64(len(vals))) == len(vals)
    for t, v in rows:
        ref.set_with_timeout(t, v, dls.get(v, 0))
    return e, ref


def _check_corpus(lib, c, how, seed=1, singles=8):
    """the light filters of corpus `c` plus _ttl_cases at NOW (the seeded deadlines lie before, at and after it), pipelined
    and in the small-graph form at capacity n + 37, then `singles` filters one at a time in the 64-filter tier"""
    rng = random.Random(seed)
    e, ref = _load(lib, c, how, NOW, rng)
    filters = c.filters(heavy=False) + _ttl_cases(ref, e, rng, NOW)
    blob, offs = pack(filters)
    want = ref.match_batch(blob, offs, NOW)
    for rows in (0, len(filters) + 37):
        rc, res, _, _ = e.match(filters, NOW, rows=rows)
        assert rc == 0, (rows, rc)
        _same(res, want, f"{how} rows={rows}")
    for q in filters[:singles]:
        rc, res, _, _ = e.match([q], NOW, rows=64)
        assert rc == 0 and res.sorted_list(0) == ref.get_message(q, NOW), q
    e.close()


def test_lookup_at_now_on_the_emulator_equals_get_message(rexp):
    """the `#` range shortcut at the root and below (edge corpus, loaded by the parallel build) and the mode-2 walk under a
    literal `#` (loaded set by set)"""
    _check_corpus(rexp, R.retained_edge_corpus(), "bulk")
    _check_corpus(rexp, R.retained_lit_hash_corpus(), "set")


def test_capacity_protocol_counts_live_handles_and_leaves_the_rest_untouched(rexp):
    e, ref = _E(rexp), TimedRetain(orc)
    for i in range(300):
        d = (NOW - 1, NOW, NOW + 1, 0)[i % 4]
        e.set(f"k/{i}", 1000 + i, d)
        ref.set_with_timeout(f"k/{i}", 1000 + i, d)
    live = ref.get_message("k/#", NOW)
    assert len(live) == 150
    for rows in (0, 64):
        rc, _, ids, needed = e.match(["k/#"], NOW, rows=rows, cap=len(live) - 1)
        assert rc == -3 and needed == len(live)
        rc, res, ids, needed = e.match(["k/#"], NOW, rows=rows, cap=len(live))
        assert rc == 0 and needed == len(live) and res.sorted_list(0) == live
        assert (ids[len(live):] == 0xEEEEEEEE).all()
    e.close()


def test_an_engine_without_deadlines_is_unaffected(rexp):
    """set_ttl with deadline 0 and a sweep leave the engine without deadlines: the lookup returns every handle"""
    e = _E(rexp)
    for i in range(50):
        e.set(f"p/{i}", i, 0)
    out = np.zeros(8, np.uint32)
    assert rexp.emu_retain_remove_expired(e.h, C.c_uint64(1 << 62), C.c_void_p(out.ctypes.data), C.c_uint64(8)) == 0
    rc, res, _, _ = e.match(["p/#"], 1 << 62)
    assert rc == 0 and res.sorted_list(0) == list(range(50))
    e.close()


def test_lookup_at_now_under_asan_ubsan(tmp_path):
    """the same kernels and host bookkeeping under AddressSanitizer + UBSan, in a subprocess (the runtime must load first)"""
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    _build(tmp_path, san=True)
    script = tmp_path / "run.py"
    script.write_text(f"""
import sys
sys.path.insert(0, {str(ROOT)!r}); sys.path.insert(0, {str(ROOT / 'tests')!r})
import _retain_edges as R
import test_retain_expiry_cpu as T
lib = T._lib({str(tmp_path / "libemu_rexp_asan.so")!r})
T._check_corpus(lib, R.retained_lit_hash_corpus(), "set", seed=2)
T.test_capacity_protocol_counts_live_handles_and_leaves_the_rest_untouched(lib)
print("asan run ok")
""")
    libasan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    env = {"PATH": "/usr/bin:/bin", "LD_PRELOAD": libasan, "ASAN_OPTIONS": "detect_leaks=0:detect_stack_use_after_return=0", "PYTHONPATH": str(ROOT)}
    import os
    import sys
    for k in ("HOME", "LD_LIBRARY_PATH", "VIRTUAL_ENV"):
        if k in os.environ:
            env[k] = os.environ[k]
    run = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600, env=env)
    assert run.returncode == 0 and "asan run ok" in run.stdout, (run.stdout[-1500:], run.stderr[-4000:])
