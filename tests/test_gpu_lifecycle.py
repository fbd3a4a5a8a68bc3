"""GPU tier: whole engine lifetimes.  In one process, several create -> use -> destroy cycles on a default engine and on a
GM_FLAG_MANUAL_FLUSH engine.  Each cycle goes through every entry point that allocates scratch, captures a graph, opens a
communicator or a fused gather, then destroys the engine with all of it in place; every result equals the oracle in every
cycle.  The oracle lists are computed once."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from rmqtt_b200 import _native as N
from rmqtt_b200 import workload as wl
from rmqtt_b200.engine import Engine, MatchResult, pack
from rmqtt_b200.router import GpuRouter, Id, SubscriptionOptions

pytestmark = pytest.mark.gpu

CYCLES = 3
CFG = wl.C2.scaled(n_subs=40_000, n_topics=6_000)
N_ROUTER = 600          # router relations, one client each; every fourth in a one-member shared group


def _canon(counts, offsets, ids):
    counts = np.asarray(counts, dtype=np.int64)
    seg = np.repeat(np.arange(len(counts)), np.maximum(counts, 0))
    ids = np.asarray(ids)[: int(offsets[-1])]
    return counts, ids[np.lexsort((ids, seg))]


def _want(res):
    return _canon(res["counts"], res["offsets"], res["ids"])


def _same(res, want, what):
    counts, ids = res.canonical()
    assert (counts == want[0]).all(), f"{what}: counts differ at {np.nonzero(counts != want[0])[0][:5]}"
    assert len(ids) == len(want[1]) and (ids == want[1]).all(), f"{what}: id multisets differ"


def _slice(blob, offs, k):
    return pack(wl.unpack(blob, offs)[:k])


@pytest.fixture(scope="module")
def data():
    sb, so, sv = wl.gen_subs(CFG)
    tb, to = wl.gen_topics(CFG)
    rb, ro, rv = wl.gen_retained(CFG, 30_000)
    fb, fo = wl.gen_retain_filters(CFG, 3_000)
    tree, rtree = orc.TopicTree(), orc.RetainTree()
    tree.bulk_insert(sb, so, sv)
    rtree.bulk_insert(rb, ro, rv)
    d = {"subs": (sb, so, sv), "retained": (rb, ro, rv)}
    # topic batches: small-graph tier 0 (<= 64 rows), tier 1 (<= 2048 rows), pipelined (more than 2048 rows)
    d["topics"] = [_slice(tb, to, 50), _slice(tb, to, 1500), (tb, to)]
    d["topics_want"] = [_want(tree.match_batch(b, o)) for b, o in d["topics"]]
    # retained filter batches: graph tiers 0 and 1, then the pipelined lookup (more than 2048 filters)
    d["filters"] = [_slice(fb, fo, 40), _slice(fb, fo, 1200), (fb, fo)]
    d["filters_want"] = [_want(rtree.match_batch(b, o)) for b, o in d["filters"]]
    # router: relation i = (filter i, client c<i>) over subscriptions that the 1500-topic batch matches; a topic's relations
    # are the oracle's ids over those filters
    assert (sv == np.arange(len(sv))).all()
    subs = wl.unpack(sb, so)
    filters = [subs[v] for v in np.unique(tree.match_batch(*d["topics"][1])["ids"])[:N_ROUTER]]
    rt = orc.TopicTree()
    for i, f in enumerate(filters):
        rt.insert(f, i)
    d["router_filters"] = [f.decode() for f in filters]
    d["router_topics"] = [t.decode() for t in wl.unpack(*d["topics"][1])]
    rtb, rto = pack(d["router_topics"])
    w = rt.match_batch(rtb, rto)
    d["router_want"] = [sorted((d["router_filters"][v], f"c{v}") for v in w["ids"][w["offsets"][i]:w["offsets"][i + 1]])
                        for i in range(len(d["router_topics"]))]
    return d


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _match_device(eng, blob, offs):
    n = len(offs) - 1
    d_blob, d_offs = torch.from_numpy(blob).cuda(), torch.from_numpy(offs.view(np.int32)).cuda()
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_needed = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_ids = torch.empty(64 * n, dtype=torch.int32, device="cuda")
    eng.match_batch_device(d_blob, d_offs, d_spans, d_ids, d_needed, d_status, _stream())
    torch.cuda.synchronize()
    m = int(d_needed.item())
    assert m <= d_ids.numel()
    return MatchResult(d_spans.cpu().numpy().view(np.uint32), d_ids.cpu().numpy().view(np.uint32), d_status.cpu().numpy(), m)


def _retain_device(eng, blob, offs, cap):
    n = len(offs) - 1
    d_blob, d_offs = torch.from_numpy(blob).cuda(), torch.from_numpy(offs.view(np.int32)).cuda()
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    d_ids = torch.zeros(max(cap, 1), dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    needed = C.c_uint64(0)
    eng._check(eng._lib.gm_retain_match_batch_device(eng._h, d_blob.data_ptr(), d_blob.numel(), d_offs.data_ptr(), n, d_spans.data_ptr(),
                                                     d_ids.data_ptr(), d_ids.numel(), C.byref(needed), d_status.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return MatchResult(d_spans.cpu().numpy().view(np.uint32), d_ids.cpu().numpy().view(np.uint32), d_status.cpu().numpy(), int(needed.value))


def _host_matches(eng, d, what):
    for k, ((b, o), want) in enumerate(zip(d["topics"], d["topics_want"])):
        _same(eng.match_batch(b, o), want, f"{what}: ids, batch {k}")
        _same(eng.match_batch_via_desc(b, o), want, f"{what}: descriptors, batch {k}")


def _retained(eng, d, what):
    for k, ((b, o), want) in enumerate(zip(d["filters"], d["filters_want"])):
        _same(eng.retain_match_batch(b, o), want, f"{what}: retained, batch {k}")
    b, o = d["filters"][1]
    _same(_retain_device(eng, b, o, len(d["filters_want"][1][1])), d["filters_want"][1], f"{what}: retained, device entry point")


def _router(manual, d, what):
    eng = Engine(manual_flush=manual)
    r = GpuRouter(eng)
    for i, f in enumerate(d["router_filters"]):
        r.add(f, Id(1, f"c{i}", i), SubscriptionOptions(shared_group=f"g{i}" if i % 4 == 0 else ""))
    for got in (r.matches_batch(d["router_topics"]), r.matches_batch_shared(d["router_topics"], seed=7)):
        for t, g, want in zip(d["router_topics"], got, d["router_want"]):   # a one-member group always chooses its member
            assert g is not None and sorted((x.topic_filter, x.client_id) for x in g) == want, (what, t)
    r._lib.gmr_destroy(r._h)         # the router goes first, then its engine
    r._h = None
    eng.close()


def _comm(eng, d, what):
    b, o = d["topics"][1]
    n = len(o) - 1
    for _ in range(2):               # a second init replaces the communicator
        eng.comm_init(Engine.comm_unique_id(), 0, 1)
    d_blob, d_offs = torch.from_numpy(b).cuda(), torch.from_numpy(o.view(np.int32)).cuda()
    d_sel = torch.zeros(n, dtype=torch.int32, device="cuda")
    k, _ = eng.partition_batch_device(d_blob, d_offs, 1, 0, d_sel, _stream())
    assert k == n
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_needed = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_ids = torch.empty(64 * n, dtype=torch.int32, device="cuda")
    eng.match_batch_device_ex(d_blob, d_offs, d_spans, d_ids, d_needed, d_status, _stream(), d_sel=d_sel, n_sel=k)
    a_idx = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    a_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    a_ids = torch.empty(64 * n, dtype=torch.int32, device="cuda")
    sizes = eng.allgatherv_device(d_sel, d_spans, k, d_ids, d_needed, a_idx, a_spans, a_ids, _stream())
    torch.cuda.synchronize()
    m = int(d_needed.item())
    assert sizes.tolist() == [[n, m]], what
    order = np.argsort(a_idx.cpu().numpy())
    _same(MatchResult(a_spans.cpu().numpy().view(np.uint32)[order], a_ids.cpu().numpy().view(np.uint32), np.zeros(n, np.int32), m),
          d["topics_want"][1], f"{what}: allgatherv")


def _gather(eng, d, what):
    b, o = d["topics"][1]
    n = len(o) - 1
    d_blob, d_offs = torch.from_numpy(b).cuda(), torch.from_numpy(o.view(np.int32)).cuda()
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    for round_ in range(2):          # created, used, destroyed; created again and used (the engine's destruction closes it)
        if round_:
            eng.gather_destroy()
        eng.gather_create(1, 0, n, 64 * n)
        eng.gather_connect([b"\0" * N.GM_IPC_HANDLE_BYTES])
        eng.match_gather_device(d_blob, d_offs, d_status, _stream())
        counts, idx, spans, ids = eng.gather_result(_stream())
        assert counts.tolist() == [[n, int(spans[:, 1].sum())]], what
        order = np.argsort(idx)
        _same(MatchResult(spans[order], ids, d_status.cpu().numpy(), int(counts[0, 1])), d["topics_want"][1], f"{what}: fused gather {round_}")


@pytest.mark.parametrize("manual", [False, True], ids=["auto_flush", "manual_flush"])
def test_create_use_destroy_cycles_equal_the_oracle(data, manual):
    sb, so, sv = data["subs"]
    rb, ro, rv = data["retained"]
    for cycle in range(CYCLES):
        what = f"{'manual' if manual else 'auto'} flush, cycle {cycle}"
        eng = Engine(manual_flush=manual, filters_hint=CFG.n_subs)
        eng.bulk_load(sb, so, sv)
        eng.retain_bulk_load(rb, ro, rv)
        if manual:
            eng.flush()
        _host_matches(eng, data, what)
        b, o = data["topics"][2]
        _same(_match_device(eng, b, o), data["topics_want"][2], f"{what}: device buffers")
        _retained(eng, data, what)
        _router(manual, data, what)
        eng.compact()                # re-ships every table: the graphs and views captured above are replaced
        _host_matches(eng, data, f"{what}, compacted")
        _retained(eng, data, f"{what}, compacted")
        _comm(eng, data, what)
        _gather(eng, data, what)
        eng.close()
