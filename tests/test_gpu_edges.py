"""GPU tier at the size boundaries of the match kernels: the corpus of tests/_edges.py (8 / 9 / 32 / 33 matched value sets,
65534 / 65535-member sets, 7 / 8 / 9 levels and deeper than the trie, 26..29-byte and long levels, wide and Bloom-colliding
nodes, batch sizes around tiles / CTAs / small-graph tiers, the tokeniser's 24 KiB stage, the small-graph text and output
capacities) through every entry point and under every scheduling knob, compared with the oracle — bit-exact sorted multisets,
status, exact work counters and the number of deferred topics.  The oracle answer of every batch is computed once; every path
is compared with it, never with another GPU run."""
import ctypes as C

import numpy as np
import pytest
import torch

import _edges as E
from rmqtt_b200 import _native as N
from rmqtt_b200 import workload as wl
from rmqtt_b200.engine import Engine, GpuMqttError, MatchResult, pack

pytestmark = pytest.mark.gpu

DEFAULT_KNOBS = dict(tok_bulk=1, sorted_rows=1, tile_chunk=1, k2_ctas=0, bucket_bits=1400, small_graphs=1, e2e_chunk=262144)
SWEEP = [{}] + [{k: v} for k, vs in (("tok_bulk", (0,)), ("sorted_rows", (0,)), ("tile_chunk", (2, 7, 1024)), ("k2_ctas", (1, 2, 3)),
                                    ("bucket_bits", (1000, 1404, 1800)), ("small_graphs", (0,))) for v in vs] + \
        [dict(tok_bulk=0, sorted_rows=0, tile_chunk=7, k2_ctas=2, bucket_bits=1404, small_graphs=0)]
BATCHES = ["main", "big_tile", "huge", "stage", "text0_at", "text0_over", "text1_at", "text1_over", "out0_at", "out0_over", "out1_at",
           "out1_over"] + [f"n{n}" for n in (1, 31, 32, 33, 64, 65, 511, 512, 513, 2048, 2049)]


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _canon(want):
    ids = want["ids"].copy()
    o = want["offsets"]
    for i in range(len(o) - 1):
        ids[o[i]:o[i + 1]].sort()
    return want["counts"], ids, o


def _select(w, rows):
    """The oracle's canonical answer for the rows `rows` of a batch."""
    counts, ids, o = w[:3]
    return counts[rows], (np.concatenate([ids[o[r]:o[r + 1]] for r in rows]) if len(rows) else ids[:0])


def _same(res, w, what, rows=None):
    wc, wi = (w[0], w[1]) if rows is None else _select(w, rows)
    counts, ids = res.canonical()
    bad = np.nonzero(counts != wc)[0]
    assert len(bad) == 0, f"{what}: counts differ at rows {bad[:5]}: {counts[bad[:5]]} vs {wc[bad[:5]]}"
    assert len(ids) == len(wi) and (ids == wi).all(), f"{what}: id multisets differ"
    assert (res.status == np.where(wc < 0, N.GM_ERR_INVALID_TOPIC, 0)).all(), f"{what}: status"


class Ctx:
    def __init__(self):
        self.c = E.subscription_corpus()
        self.trees = self.c.tree_oracles()
        E.check_against_oracle(self.c, self.trees[0])
        self.eng = Engine(device=0)
        self.c.load_engine(self.eng)
        self.want = {}
        self.packed = {}
        for name in BATCHES:
            tb, to = self.c.packed(name)
            self.packed[name] = (tb, to)
            want = self.trees[0].match_batch(tb, to)
            self.want[name] = (*_canon(want), want["counters"])

    def reset(self):
        for k, v in DEFAULT_KNOBS.items():
            self.eng.debug_knob(k, v)


@pytest.fixture(scope="module")
def ctx():
    x = Ctx()
    yield x
    x.eng.close()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _to_dev(tb, to, shift=0):
    """The blob at `shift` bytes past a 16-byte boundary (the tokeniser then cannot stage it)."""
    raw = torch.zeros(len(tb) + 64, dtype=torch.uint8, device="cuda")
    base = (16 - raw.data_ptr() % 16) % 16
    d_blob = raw[base + shift:base + shift + len(tb)]
    assert d_blob.data_ptr() % 16 == shift
    if len(tb):
        d_blob.copy_(torch.from_numpy(tb))
    return d_blob, torch.from_numpy(to.view(np.int32)).cuda()


def _device(eng, tb, to, total, shift=0, work=False):
    n = len(to) - 1
    d_blob, d_offs = _to_dev(tb, to, shift)
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    d_ids = torch.zeros(max(1, total), dtype=torch.int32, device="cuda")
    d_needed = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    w = eng.match_batch_device(d_blob, d_offs, d_spans, d_ids, d_needed, d_status, _stream(), work=work)
    torch.cuda.synchronize()
    assert int(d_needed.item()) == total
    return MatchResult(d_spans.cpu().numpy().view(np.uint32), d_ids.cpu().numpy().view(np.uint32), d_status.cpu().numpy(), total), w


def _expand(eng, spans, descs, status):
    """Descriptor-mode output -> MatchResult of ids (the expansion Engine.match_batch_via_desc does)."""
    _, rng, _ = eng.values_view()
    cnt = descs[:, 1].astype(np.int64)
    big = cnt == E.CNT_BIG
    cnt[big] = rng[descs[big, 0], 1]
    starts = np.zeros(len(descs) + 1, dtype=np.int64)
    np.cumsum(cnt, out=starts[1:])
    ids = eng.desc_expand(descs) if len(descs) else np.zeros(0, np.uint32)
    d0 = spans[:, 0].astype(np.int64)
    d1 = d0 + spans[:, 1].astype(np.int64)
    return MatchResult(np.stack([starts[d0], starts[d1] - starts[d0]], axis=1).astype(np.uint32), ids, status, len(ids))


def _device_ex(eng, tb, to, rows, cap, desc):
    d_blob, d_offs = _to_dev(tb, to)
    n = len(rows)
    d_sel = torch.from_numpy(rows.astype(np.int32)).cuda()
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    d_out = torch.zeros((max(1, cap), 2) if desc else max(1, cap), dtype=torch.int32, device="cuda")
    d_needed = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    eng.match_batch_device_ex(d_blob, d_offs, d_spans, d_out, d_needed, d_status, _stream(), desc=desc, d_sel=d_sel, n_sel=n)
    torch.cuda.synchronize()
    needed = int(d_needed.item())
    assert needed == cap, (needed, cap)
    spans, status = d_spans.cpu().numpy().view(np.uint32), d_status.cpu().numpy()
    if desc:
        return _expand(eng, spans, d_out.cpu().numpy().view(np.uint32).reshape(-1, 2)[:needed], status)
    return MatchResult(spans, d_out.cpu().numpy().view(np.uint32), status, needed)


def _check_batch(x, name, full):
    """Every entry point on one batch; `full` adds the unaligned-blob, gather and instrumented variants."""
    eng, c = x.eng, x.c
    tb, to = x.packed[name]
    w = x.want[name]
    total = int(w[0].clip(0).sum())
    n = len(to) - 1
    _same(eng.match_batch(tb, to), w, f"{name} gm_match_batch")
    _same(eng.match_batch_via_desc(tb, to), w, f"{name} gm_match_batch_desc")
    _same(_device(eng, tb, to, total)[0], w, f"{name} gm_match_batch_device")
    rows = np.random.default_rng(n).permutation(n)[:max(1, (3 * n) // 4)]
    cases = c.batches[name]
    _same(_device_ex(eng, tb, to, rows, int(w[0][rows].clip(0).sum()), False), w, f"{name} device_ex ids", rows)
    _same(_device_ex(eng, tb, to, rows, sum(cases[r].F or 0 for r in rows), True), w, f"{name} device_ex descriptors", rows)
    res, work = _device(eng, tb, to, total, work=True)                  # instrumented kernels: exact work counters
    _same(res, w, f"{name} instrumented")
    k = w[3]
    assert (work["visited"], work["probed"], work["filters"], work["ids"]) == (k["V"], k["E"], k["F"], k["M"]), name
    assert work["deferred"] == c.n_deferred(name), name
    if not full:
        return
    shift = 1 + n % 15
    _same(_device(eng, tb, to, total, shift=shift)[0], w, f"{name} device, blob {shift} bytes past 16")
    eng.gather_create(1, 0, n, total + 16)                              # the fused gather at world 1
    try:
        eng.gather_connect([b"\0" * N.GM_IPC_HANDLE_BYTES])
        d_blob, d_offs = _to_dev(tb, to)
        d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
        eng.match_gather_device(d_blob, d_offs, d_status, _stream())
        counts, idx, spans, ids = eng.gather_result(_stream())
        assert counts.tolist() == [[n, total]]
        order = np.argsort(idx)
        assert (idx[order] == np.arange(n)).all()
        _same(MatchResult(spans[order], ids, d_status.cpu().numpy(), total), w, f"{name} gather")
    finally:
        eng.gather_destroy()


@pytest.mark.parametrize("knobs", SWEEP, ids=lambda k: "-".join(f"{a}={b}" for a, b in k.items()) or "defaults")
def test_corpus_every_entry_point_under_every_knob(ctx, knobs):
    """`debug_knob` promises that no scheduling knob changes a result: one knob at a time off its default, then all of them."""
    ctx.reset()
    try:
        for k, v in knobs.items():
            ctx.eng.debug_knob(k, v)
        for name in BATCHES:
            _check_batch(ctx, name, full=not knobs or len(knobs) > 1)
    finally:
        ctx.reset()


def test_extra_tree_rows(ctx):
    tb, to = ctx.packed["main"]
    cases = ctx.c.batches["main"]
    rows = np.asarray([(0, 1, 5, 9)[i % 4] for i in range(len(cases))], dtype=np.uint32)      # tree 9 does not exist
    for small in (1, 0):
        ctx.eng.debug_knob("small_graphs", small)
        res = ctx.eng.match_batch_trees(tb, to, rows)
        for i, x in enumerate(cases):
            tr = int(rows[i])
            want = None if x.F is None else sorted(ctx.trees[tr].matches(x.topic)) if tr in ctx.trees else []
            assert res.sorted_list(i) == want, (x.topic, tr)
    ctx.reset()


def _raw(eng, tb, to, cap, desc=False):
    """gm_match_batch / gm_match_batch_desc with an exact capacity -> (rc, needed, MatchResult in ids)."""
    n = len(to) - 1
    spans = np.zeros((n, 2), dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    out = np.zeros((max(cap, 1), 2) if desc else max(cap, 1), dtype=np.uint32)
    needed = C.c_uint64(0)
    fn = eng._lib.gm_match_batch_desc if desc else eng._lib.gm_match_batch
    rc = fn(eng._h, _vp(tb), _vp(to), n, _vp(spans), _vp(out), cap, C.byref(needed), _vp(status))
    if rc != N.GM_OK:
        return rc, int(needed.value), None
    return rc, int(needed.value), _expand(eng, spans, out[:int(needed.value)], status) if desc else MatchResult(spans, out, status, int(needed.value))


def _capacity_edge(eng, tb, to, w, n_desc, what):
    total = int(w[0].clip(0).sum())
    for desc, need in ((False, total), (True, n_desc)):
        rc, needed, res = _raw(eng, tb, to, need, desc)
        assert rc == N.GM_OK and needed == need, (what, desc, rc, needed, need)
        _same(res, w, f"{what} cap = needed (desc={desc})")
        if need:
            rc, needed, _ = _raw(eng, tb, to, need - 1, desc)
            assert rc == N.GM_ERR_CAPACITY and needed == need, (what, desc, rc, needed, need)


def test_capacity_protocol_at_the_exact_edge(ctx):
    """cap = needed succeeds, cap = needed - 1 is GM_ERR_CAPACITY with the right `needed`, in ids and descriptors: both
    small-graph tiers, the single-chunk and the multi-chunk pipelined host path (chunks of 1024 topics that start at
    unaligned text offsets)."""
    eng, c = ctx.eng, ctx.c
    for name in ("n1", "n64", "n2048", "n2049", "out0_over", "text1_over"):
        tb, to = ctx.packed[name]
        _capacity_edge(eng, tb, to, ctx.want[name], sum(x.F or 0 for x in c.batches[name]), name)
    main = c.batches["main"]
    cases = [main[(i * 11) % len(main)] for i in range(5000)]
    tb, to = pack([x.topic for x in cases])
    assert [int(to[k]) % 16 for k in (1024, 2048, 3072, 4096)].count(0) == 0, "chunk boundaries at unaligned text offsets"
    want = ctx.trees[0].match_batch(tb, to)
    n_desc = sum(x.F or 0 for x in cases)
    assert want["counters"]["F"] == n_desc
    w = _canon(want)
    eng.debug_knob("e2e_chunk", 1024)
    try:
        _same(eng.match_batch(tb, to), w, "5 chunks")
        _same(eng.match_batch_via_desc(tb, to), w, "5 chunks, descriptors")
        _capacity_edge(eng, tb, to, w, n_desc, "5 chunks")
    finally:
        ctx.reset()


def test_small_graph_tiers_at_their_text_and_output_capacities():
    """A batch exactly at a tier's text / output capacity runs as that tier's graph; one byte or one id more falls back (to
    the next tier or the pipelined path) — and every one of them is still exact.  Which path ran shows in the kernel timing
    ring: only the pipelined path records it."""
    c = E.subscription_corpus()
    eng, tree = Engine(device=0), E.orc.TopicTree()
    for f, v in c.adds:
        if f.startswith(("stage/", "outs/")) or (f, v) in E.ROOT_WILD:
            eng.add(f, v)
            tree.insert(f, v)
    for name, tier, pipelined in (("text0_at", 0, False), ("text0_over", 1, False), ("text1_at", 1, False), ("text1_over", None, True),
                                  ("out0_at", 0, False), ("out0_over", None, True), ("out1_at", 1, False), ("out1_over", None, True)):
        cap_n, cap_blob, cap_out = E.SMALL_TIERS[0 if name.endswith("0_at") or name.endswith("0_over") else 1]
        tb, to = c.packed(name)
        n = len(to) - 1
        w = _canon(tree.match_batch(tb, to))
        total = int(w[0].clip(0).sum())
        assert n <= cap_n
        if name.startswith("text"):
            assert int(to[-1]) == cap_blob + name.endswith("_over")
        else:
            assert int(to[-1]) <= cap_blob and total == cap_out + name.endswith("_over")
        ring = len(eng.kernel_ms())
        _same(eng.match_batch(tb, to), w, name)
        assert (len(eng.kernel_ms()) > ring) == pipelined, name
        _same(eng.match_batch_via_desc(tb, to), w, name + " descriptors")
    eng.close()


def test_second_engine_with_tiny_windows_wide_nodes_and_a_shallow_trie(monkeypatch):
    """8-slot windows (probes wrap, the tables re-hash), a node with more than WIDE_FANOUT children, a saturated Bloom mask probed
    with tokens that are no child of it; 12-level topics stay on the fast path because the trie is 3 levels deep."""
    monkeypatch.setenv("GM_WIN_MIN_SLOTS_LOG2", "3")
    s = E.subscription_corpus(shallow=True)
    eng = Engine(device=0)
    s.load_engine(eng)
    tree = s.load_oracle()
    E.check_against_oracle(s, tree)
    tb, to = s.packed("main")
    want = tree.match_batch(tb, to)
    w = _canon(want)
    total = int(w[0].clip(0).sum())
    _same(eng.match_batch(tb, to), w, "host")
    _same(eng.match_batch_via_desc(tb, to), w, "descriptors")
    res, work = _device(eng, tb, to, total, work=True)
    _same(res, w, "instrumented")
    k = want["counters"]
    assert (work["visited"], work["probed"], work["filters"], work["ids"], work["deferred"]) == (k["V"], k["E"], k["F"], k["M"], 0)
    assert sum(work["misses_by_depth"]) > 0                             # some literal probes passed the Bloom mask and missed
    eng.close()


def test_c3_shaped_work_counters():
    """C3-shaped data (64-way fan-out at the top: wide nodes, several windows, populated locality buckets) through the
    instrumented device entry point: V / E / F / M equal the oracle's."""
    cfg = wl.C3.scaled(n_subs=2_000_000, n_topics=200_000)
    sb, so, sv = wl.gen_subs(cfg)
    tb, to = wl.gen_topics(cfg)
    eng, tree = Engine(device=0, filters_hint=cfg.n_subs), E.orc.TopicTree()
    assert eng.bulk_load(sb, so, sv) == tree.bulk_insert(sb, so, sv, nthreads=8)
    want = tree.match_batch(tb, to, nthreads=8)
    w = _canon(want)
    res, work = _device(eng, tb, to, int(w[0].clip(0).sum()), work=True)
    _same(res, w, "C3")
    k = want["counters"]
    assert (work["visited"], work["probed"], work["filters"], work["ids"]) == (k["V"], k["E"], k["F"], k["M"])
    eng.close()


def test_retained_lookup_deep_shadowing_and_a_scratch_that_must_grow():
    """The retained corpus (levels beyond the 8-level token row, literal '+' / '#' levels that shadow wildcard expansion, `$`
    roots, removals) on the device; then again from a 64-item scratch: the lookup must grow it (more than one attempt's
    launches) and still be exact."""
    ops, filters = E.retained_corpus()
    eng = Engine(device=0)

    def put(t, v):
        try:
            eng.retain_set(t, v)
            return True
        except GpuMqttError:
            return False

    def rm(t):
        try:
            return eng.retain_remove(t) is not None
        except GpuMqttError:
            return False

    rt = E.load_retained(ops, put, rm)
    fb, fo = pack(filters)
    w = _canon(rt.match_batch(fb, fo))
    _same(eng.retain_match_batch(fb, fo), w, "retained")               # (ships the tree)
    l0 = eng.kernel_launches()
    _same(eng.retain_match_batch(fb, fo), w, "retained, again")
    one = eng.kernel_launches() - l0                                      # one attempt of the default-sized scratch
    with pytest.raises(GpuMqttError):
        eng.debug_knob("retain_caps", 100)                                # not a multiple of 64
    eng.debug_knob("retain_caps", 64)
    l0 = eng.kernel_launches()
    _same(eng.retain_match_batch(fb, fo), w, "retained, grown scratch")
    grown = eng.kernel_launches() - l0
    assert grown > one and grown % one == 0, (grown, one)
    eng.close()
