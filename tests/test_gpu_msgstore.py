"""GPU tier of the message store (gm_msgstore_*) through the real ABI: every case of tests/_msgstore_cases.py, a seeded
differential against tests/_msgstore_oracle.py on a C4-shaped store of 200 K messages with 20 K-filter batches, a 5 000-query
batch of one client, and the retained lookup of a plain engine, which the store's entry point must leave unchanged."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

import _msgstore_cases as K
from _msgstore_oracle import MsgStoreRef
from oracle import oracle as orc
from rmqtt_b200 import _native as N
from rmqtt_b200 import workload as wl
from rmqtt_b200.engine import Engine, pack
from rmqtt_b200.msgstore import GpuMessageStore

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

NOW = K.NOW


class GpuStore:
    """the adapter of _msgstore_cases over GpuMessageStore"""

    def __init__(self, initial_mark_slots=0):
        self.eng = Engine(max_levels=16)
        self.ms = GpuMessageStore(self.eng, initial_mark_slots=initial_mark_slots)

    def close(self):
        self.ms.close()
        self.eng.close()

    def store(self, topic, h, expiry, fwd):
        self.ms.store(topic, h, expiry, fwd)

    def get(self, now, filters, clients, groups, cap=None):
        n = len(filters)
        blob, offs = pack(filters)
        cl = np.array([self.ms.client_key(c) for c in clients], np.uint32)
        sh = np.array([self.ms.share_key(f, g) for f, g in zip(filters, groups)], np.uint32)
        c = cap if cap is not None else 16 * n + 1024
        spans, status, out = np.zeros((n, 2), np.uint32), np.zeros(n, np.int32), np.empty(max(c, 1), np.uint32)
        needed = C.c_uint64(0)
        rc = N.lib().gm_msgstore_get_batch(self.ms._h, int(now), blob.ctypes.data, offs.ctypes.data, n, cl.ctypes.data, sh.ctypes.data, spans.ctypes.data,
                                           out.ctypes.data, c, C.byref(needed), status.ctypes.data)
        if cap is None and rc == N.GM_ERR_CAPACITY:
            return self.get(now, filters, clients, groups, int(needed.value))
        if rc != 0:
            return rc, int(needed.value), None
        return 0, int(needed.value), [None if status[i] else sorted(out[spans[i, 0]:spans[i, 0] + spans[i, 1]].tolist()) for i in range(n)]

    def remove_expired(self, now, cap):
        return self.ms.remove_expired(now, cap).tolist()

    def stats(self):
        return self.ms.stats()


@pytest.mark.parametrize("case", K.ALL, ids=[c.__name__ for c in K.ALL])
def test_cases(case):
    S, ref = GpuStore(initial_mark_slots=64), MsgStoreRef(orc)
    case(S, ref)
    S.close()


def test_seeded_rounds_small():
    S, ref = GpuStore(initial_mark_slots=64), MsgStoreRef(orc)
    K.random_rounds(S, ref, 21, rounds=8, per_round=200, batch=800, n_clients=40, n_groups=5)
    S.close()


def _c4_store(n_msgs, rng, marked=0.1, n_clients=2000):
    blob, offs, handles = wl.gen_retained(wl.C4, n_msgs)
    topics = [t.decode() for t in wl.unpack(blob, offs)]
    expiry = [NOW + rng.randrange(-2_000, 60_000) for _ in range(n_msgs)]
    fwd = [[(f"c{rng.randrange(n_clients)}", None)] if rng.random() < marked else [] for _ in range(n_msgs)]
    S, ref = GpuStore(), MsgStoreRef(orc)
    S.ms.store_batch(topics, handles, expiry, fwd)
    for t, h, e, f in zip(topics, handles.tolist(), expiry, fwd):
        ref.set(t, h, e, f)
    return S, ref, n_msgs


def test_c4_seeded_differential():
    """200 K C4 messages with store-time marks; rounds of 20 K-filter batches from repeated clients and shared groups (filters
    drawn from a pool, so that (filter, group) pairs repeat too), new messages stored with marks, and sweeps as now advances"""
    rng = random.Random(4)
    S, ref, h = _c4_store(200_000, rng)
    fb, fo = wl.gen_retain_filters(wl.C4, 20_000)
    pool = [f.decode() for f in wl.unpack(fb, fo)][:4000]
    now = NOW
    for rnd in range(3):
        q = [(rng.choice(pool), f"c{rng.randrange(2000)}", None if rng.random() < 0.7 else f"g{rng.randrange(3)}") for _ in range(20_000)]
        got = K.check(S, ref, now, q)
        assert sum(len(g) for g in got if g) > 1000
        for _ in range(2000):
            t = rng.choice(pool).replace("+", "x").replace("#", "y")
            K.put(S, ref, t, h, expiry=now + rng.randrange(0, 5000), fwd=[(f"c{rng.randrange(2000)}", None)])
            h += 1
        now += 700
        assert sorted(S.remove_expired(now, 1 << 20)) == sorted(ref.remove_expired(now))
    st = S.stats()
    assert st["mark_slots"] >= 2 * st["marks"] and st["messages"] == len(ref.expiry)
    S.close()


def test_one_client_5000_queries():
    rng = random.Random(6)
    S, ref, _ = _c4_store(50_000, rng, marked=0.0)
    fb, fo = wl.gen_retain_filters(wl.C4, 5000)
    q = [(f.decode(), "solo", None) for f in wl.unpack(fb, fo)]
    q[:200] = [("#", "solo", None)] + q[1:200]
    got = K.check(S, ref, NOW, q)
    assert sum(len(g) for g in got if g) > 0
    assert K.check(S, ref, NOW, q) == [[] if g is not None else None for g in got]
    S.close()


def test_plain_engine_retained_lookup_is_unchanged():
    """gm_retain_match_batch_device_at on an engine without a store: the oracle's results at several now values"""
    from _retain_expiry import TimedRetain
    rng = random.Random(9)
    blob, offs, vals = wl.gen_retained(wl.C4, 100_000)
    eng, ref = Engine(), TimedRetain(orc)
    dl = np.array([0 if rng.random() < 0.5 else NOW + rng.randrange(-500, 500) for _ in range(len(vals))], np.uint64)
    eng.retain_bulk_load(blob, offs, vals, dl)
    for t, v, d in zip(wl.unpack(blob, offs), vals.tolist(), dl.tolist()):
        ref.set_with_timeout(t, v, d)
    fb, fo = wl.gen_retain_filters(wl.C4, 4096)
    fb = np.concatenate([fb, np.frombuffer(b"#", np.uint8)])
    fo = np.concatenate([fo, [fo[-1] + 1]]).astype(np.uint32)
    n = len(fo) - 1
    dev = torch.device("cuda")
    d_blob = torch.from_numpy(np.concatenate([fb, np.zeros(16, np.uint8)])).to(dev)
    d_offs = torch.from_numpy(fo.view(np.int32)).to(dev)
    lib = N.lib()
    for now in (NOW - 1000, NOW, NOW + 1000):
        want = ref.match_batch(fb, fo, now)
        cap = int(want["offsets"][-1]) + 16
        d_spans = torch.zeros((n, 2), dtype=torch.int32, device=dev)
        d_ids = torch.zeros(cap, dtype=torch.int32, device=dev)
        d_status = torch.zeros(n, dtype=torch.int32, device=dev)
        needed = C.c_uint64(0)
        s = torch.cuda.current_stream().cuda_stream
        assert lib.gm_retain_match_batch_device_at(eng._h, now, d_blob.data_ptr(), len(fb), d_offs.data_ptr(), n, d_spans.data_ptr(), d_ids.data_ptr(), cap,
                                                   C.byref(needed), d_status.data_ptr(), s) == 0
        torch.cuda.synchronize()
        spans, ids, status = d_spans.cpu().numpy().view(np.uint32), d_ids.cpu().numpy().view(np.uint32), d_status.cpu().numpy()
        assert needed.value == int(want["offsets"][-1])
        for i in range(n):
            assert (status[i] == 0) == (want["counts"][i] >= 0)
            got = np.sort(ids[spans[i, 0]:spans[i, 0] + spans[i, 1]])
            assert got.tolist() == want["ids"][int(want["offsets"][i]):int(want["offsets"][i + 1])].tolist()
    eng.close()
