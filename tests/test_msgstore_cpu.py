"""CPU tier of the message store (gm_msgstore_*).

* The host bookkeeping on a GM_FLAG_HOST_ONLY engine through the real ABI: the key a message is kept under, last-wins
  de-duplication of store-time marks, the sweep at now (expiry_time_at <= now), eviction order with now = UINT64_MAX - 1,
  retired handles, and the argument checks.
* The store's host logic and kernels (msgstore.cuh) on the CPU emulation (tests/native/emu/emu_msgstore.cpp), plain and under
  ASan + UBSan, on poisoned scratch with guarded outputs: every case of tests/_msgstore_cases.py and a seeded differential
  against tests/_msgstore_oracle.py's restatement of rmqtt-message-storage's RAM backend."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import _msgstore_cases as K
from _msgstore_oracle import MsgStoreRef
from oracle import oracle as orc
from rmqtt_b200 import _native as N
from rmqtt_b200.engine import Engine, GpuMqttError, pack
from rmqtt_b200.msgstore import NO_SHARE, GpuMessageStore
from test_emu_kernels import CSRC, EMU, ROOT

NOW = K.NOW
U64_MAX = (1 << 64) - 1


# ---- bookkeeping on a host-only engine -------------------------------------------------------------------------------
def _host_store(**kw):
    eng = Engine(host_only=True, max_levels=9)
    return eng, GpuMessageStore(eng, **kw)


def test_a_message_is_kept_under_topic_slash_handle():
    eng, ms = _host_store()
    ms.store("a/b", 7, NOW)
    ms.store("", 8, NOW)
    assert eng.stats()["retained_values"] == 2 and ms.stats()["messages"] == 2
    assert eng.retain_remove("a/b/7") == 7
    assert eng.retain_remove("/8") == 8


def test_store_time_marks_last_entry_per_client_wins():
    _, ms = _host_store()
    ms.store("t", 1, NOW, [("A", ("t/#", "g")), ("A", None), ("B", ("t/#", "g")), ("B", ("t/#", "h"))])
    # A -> None (client entry only), B -> (t/#, h) (client entry + share entry)
    assert ms.stats()["pending_marks"] == 3
    ms.store("t", 2, NOW, [("A", None), ("A", ("t/#", "g"))])
    assert ms.stats()["pending_marks"] == 5


def test_sweep_removes_at_expiry_time_and_evicts_earliest_first():
    _, ms = _host_store()
    for h, e in ((1, NOW - 1), (2, NOW), (3, NOW + 1), (4, NOW + 5), (5, NOW + 2)):
        ms.store(f"s/{h}", h, e)
    assert sorted(ms.remove_expired(NOW - 2).tolist()) == []
    assert sorted(ms.remove_expired(NOW).tolist()) == [1, 2]            # expiry_time_at <= now (ram.rs:159)
    assert ms.remove_expired(U64_MAX - 1, 2).tolist() == [3, 5]         # eviction: earliest expiry first
    assert ms.stats()["messages"] == 1
    assert ms.remove_expired(U64_MAX - 1, 0).tolist() == []
    assert ms.remove_expired(U64_MAX, 5).tolist() == [4]


def test_retired_handles_and_reuse():
    _, ms = _host_store()
    ms.store("r", 9, NOW, [("A", None)])
    with pytest.raises(GpuMqttError) as ei:
        ms.store("r2", 9, NOW)                                          # stored once while live
    assert ei.value.code == N.GM_ERR_INVALID_ARG
    assert ms.remove_expired(NOW).tolist() == [9]
    st = ms.stats()
    assert st["retired"] == 1 and st["messages"] == 0 and st["pending_marks"] == 0   # its store-time marks went with it
    ms.store("r2", 9, NOW + 10, [("B", None)])
    assert ms.stats()["retired"] == 1 and ms.stats()["pending_marks"] == 1
    ms.remove_expired(NOW + 10)
    assert ms.stats()["retired"] == 1                                  # counted once


def test_argument_checks():
    eng, ms = _host_store()
    for call in (lambda: ms.store("x", 1 << 28, NOW), lambda: ms.store("x", 1, U64_MAX)):
        with pytest.raises(GpuMqttError) as ei:
            call()
        assert ei.value.code == N.GM_ERR_INVALID_ARG
    lib, h = N.lib(), ms._h
    cl = np.array([1 << 31], np.uint32)
    assert lib.gm_msgstore_store(h, b"x", 1, 1, NOW, cl.ctypes.data, None, 1) == N.GM_ERR_INVALID_ARG
    with pytest.raises(GpuMqttError) as ei:
        ms.store("a/#/x", 2, NOW)
    assert ei.value.code == N.GM_ERR_INVALID_TOPIC
    with pytest.raises(GpuMqttError) as ei:
        ms.store_batch(["b/1", "b/#", "b/2"], [3, 4, 5], [NOW] * 3)
    assert ei.value.code == N.GM_ERR_INVALID_TOPIC
    assert eng.stats()["retained_values"] == 0 and ms.stats()["messages"] == 0     # nothing of the refused batch stays
    ms.store_batch(["b/1", "b/2"], [3, 4], [NOW, NOW + 1], [[("A", None)], []])
    assert ms.stats()["messages"] == 2 and ms.stats()["pending_marks"] == 1
    with pytest.raises(GpuMqttError) as ei:
        ms.get_batch(NOW, ["b/+"], ["A"])
    assert ei.value.code == N.GM_ERR_NO_DEVICE
    cfg = N.GmMsgstoreConfig(C.sizeof(N.GmMsgstoreConfig), 100)
    out = C.c_void_p()
    assert lib.gm_msgstore_create(eng._h, C.byref(cfg), C.byref(out)) == N.GM_ERR_INVALID_ARG


# ---- the store on the CPU emulation ----------------------------------------------------------------------------------
def _build(tmp, san: bool):
    out = tmp / ("libemu_ms_asan.so" if san else "libemu_ms.so")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-DGM_CPU_EMU", f"-I{EMU}", f"-I{CSRC}", "-shared", "-fPIC", "-pthread", "-fno-omit-frame-pointer",
           *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"] if san else []),
           "-o", str(out), str(EMU / "emu_msgstore.cpp"), str(CSRC / "host_trie.cpp"), str(CSRC / "retain_tree.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr and "cannot find" in r.stderr:
        pytest.skip("sanitizer runtime not installed")
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _lib(path):
    lib = C.CDLL(str(path))
    lib.emu_ms_new.restype = C.c_void_p
    lib.emu_ms_new.argtypes = [C.c_uint32]
    lib.emu_ms_free.argtypes = [C.c_void_p]
    lib.emu_ms_error.restype = C.c_char_p
    lib.emu_ms_store.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.emu_ms_store_batch.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64] + [C.c_void_p] * 3
    lib.emu_ms_get_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                     C.POINTER(C.c_uint64), C.c_void_p]
    lib.emu_ms_remove_expired.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.emu_ms_stats.argtypes = [C.c_void_p, C.POINTER(N.GmMsgstoreStats)]
    return lib


GUARD = 64
POISON = 0x5A5A5A5A


class EmuStore:
    """the adapter of _msgstore_cases over the emulated store; outputs carry guard words that must survive"""

    def __init__(self, lib, initial_mark_slots=0):
        self.lib, self.h = lib, C.c_void_p(lib.emu_ms_new(initial_mark_slots))
        self.clients, self.shares = {}, {}

    def close(self):
        self.lib.emu_ms_free(self.h)

    def ck(self, c):
        return self.clients.setdefault(c, len(self.clients))

    def sk(self, f, g):
        return NO_SHARE if g is None else self.shares.setdefault((f, g), len(self.shares))

    def store(self, topic, h, expiry, fwd):
        cl = np.array([self.ck(c) for c, _ in fwd], np.uint32)
        sh = np.array([NO_SHARE if s is None else self.sk(*s) for _, s in fwd], np.uint32)
        b = topic.encode()
        rc = self.lib.emu_ms_store(self.h, b, len(b), h, expiry, cl.ctypes.data, sh.ctypes.data, len(cl))
        assert rc == 0, (rc, self.lib.emu_ms_error())

    def get(self, now, filters, clients, groups, cap=None):
        n = len(filters)
        blob, offs = pack(filters)
        cl = np.array([self.ck(c) for c in clients], np.uint32)
        sh = np.array([self.sk(f, g) for f, g in zip(filters, groups)], np.uint32)
        c = cap if cap is not None else 64 * n + 64
        spans = np.full((n + GUARD, 2), POISON, np.uint32)
        status = np.full(n + GUARD, POISON, np.int32)
        out = np.full(c + GUARD, POISON, np.uint32)
        needed = C.c_uint64(0)
        rc = self.lib.emu_ms_get_batch(self.h, now, blob.ctypes.data, offs.ctypes.data, n, cl.ctypes.data, sh.ctypes.data, spans.ctypes.data, out.ctypes.data, c,
                                       C.byref(needed), status.ctypes.data)
        assert rc != -60, "a launch wrote past a scratch block"
        assert (spans[n:] == POISON).all() and (status[n:] == POISON).all() and (out[c:] == POISON).all(), "a write past an output"
        if cap is None and rc == N.GM_ERR_CAPACITY:
            return self.get(now, filters, clients, groups, int(needed.value))
        if rc != 0:
            return rc, int(needed.value), None
        lists = [None if status[i] != 0 else sorted(out[spans[i, 0]:spans[i, 0] + spans[i, 1]].tolist()) for i in range(n)]
        return rc, int(needed.value), lists

    def remove_expired(self, now, cap):
        out = np.full(cap + GUARD, POISON, np.uint32)
        n = C.c_uint64(0)
        assert self.lib.emu_ms_remove_expired(self.h, now, out.ctypes.data, cap, C.byref(n)) == 0
        assert (out[cap:] == POISON).all()
        return out[:n.value].tolist()

    def stats(self):
        s = N.GmMsgstoreStats()
        assert self.lib.emu_ms_stats(self.h, C.byref(s)) == 0
        return s.as_dict()


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _lib(_build(tmp_path_factory.mktemp("ems"), san=False))


def run_cases(lib, big_group=1000):
    for case in K.ALL:
        S, ref = EmuStore(lib, initial_mark_slots=64), MsgStoreRef(orc)
        if case is K.case_big_group:
            case(S, ref, members=big_group)
        else:
            case(S, ref)
        S.close()


def run_random(lib, seed, rounds=6):
    S, ref = EmuStore(lib, initial_mark_slots=64), MsgStoreRef(orc)
    K.random_rounds(S, ref, seed, rounds=rounds, per_round=60, batch=120, n_clients=25, n_groups=4)
    st = S.stats()
    S.close()
    return st


def test_cases_on_the_emulation(emu):
    run_cases(emu)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_seeded_differential_on_the_emulation(emu, seed):
    st = run_random(emu, seed)
    assert st["rehashes"] >= 1


def test_cases_under_asan_ubsan(tmp_path):
    so = _build(tmp_path, san=True)
    script = tmp_path / "run.py"
    script.write_text(f"""
import sys
sys.path.insert(0, {str(ROOT)!r}); sys.path.insert(0, {str(ROOT / 'tests')!r})
import test_msgstore_cpu as T
lib = T._lib({str(so)!r})
T.run_cases(lib, big_group=200)
T.run_random(lib, 7, rounds=3)
print("asan run ok")
""")
    libasan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    env = {"PATH": "/usr/bin:/bin", "LD_PRELOAD": libasan, "ASAN_OPTIONS": "detect_leaks=0:detect_stack_use_after_return=0", "PYTHONPATH": str(ROOT)}
    for k in ("HOME", "LD_LIBRARY_PATH", "VIRTUAL_ENV"):
        if k in os.environ:
            env[k] = os.environ[k]
    run = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=1500, env=env)
    assert run.returncode == 0 and "asan run ok" in run.stdout, (run.stdout[-1500:], run.stderr[-4000:])
