"""GPU tier: the CUDA path (through the C ABI) against the CPU oracle — bit-exact sorted multisets.

Every test calls gm_match_batch / gm_match_batch_device in libgpumqtt.so; nothing here can pass on a
fallback because there is none (the library refuses to match without a CUDA device)."""
import random

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from rmqtt_b200 import _native as N
from rmqtt_b200 import workload as wl
from rmqtt_b200.engine import Engine, GpuMqttError, pack

from _gen import rand_filter, rand_topic

pytestmark = pytest.mark.gpu


def _canon_oracle(want):
    ids = want["ids"].copy()
    o = want["offsets"]
    for i in range(len(o) - 1):
        ids[o[i]:o[i + 1]].sort()
    return want["counts"], ids


def _assert_same(res, want):
    counts, ids = res.canonical()
    wc, wi = _canon_oracle(want)
    assert (counts == wc).all(), f"counts differ at {np.nonzero(counts != wc)[0][:5]}"
    assert (ids == wi).all()


def test_golden_trie_rs_417_449(golden):
    g = golden["trie_A1"]
    eng = Engine()
    for f, v in g["inserts"]:
        eng.add(f, v)
    for topic, want in g["matches"]:
        assert eng.matches(topic) == sorted(want), topic
    for topic, bad in g["not_matches"]:
        assert eng.matches(topic) != sorted(bad)
    for f, v, want in g["removes"]:
        assert eng.remove(f, v) is want
    for topic, want in g["after_remove_matches"]:
        assert eng.matches(topic) == sorted(want), topic


def test_golden_trie_rs_452_498(golden):
    g = golden["trie_A2"]
    eng = Engine()
    for f, v in g["inserts"]:
        eng.add(f, v)
    r = g["range_inserts"]
    for v in range(r["lo"], r["hi"]):
        eng.add(r["pattern_each"].format(v=v), v)
    for v in range(r["lo"], r["hi"]):
        eng.add(r["pattern_same"], v)
    assert eng.stats()["values"] == 7 + 9999 - 2 + 9999
    for topic, want in g["matches"]:
        assert eng.matches(topic) == sorted(want), topic
    assert eng.matches("/iot/x") == sorted(list(range(1, 10000)) + [3])     # 10 000 ids: deferred (slow) path
    for f, v in g["stage2_inserts"]:
        eng.add(f, v)
    for topic, want in g["stage2_matches"]:
        assert eng.matches(topic) == sorted(want), topic
    for f, v in g["stage3_inserts"]:
        eng.add(f, v)
    for topic, want in g["stage3_matches"]:
        assert eng.matches(topic) == sorted(want), topic


def test_golden_derived_dollar_and_literal_wildcards(golden):
    g = golden["derived_A5"]["trie"]
    eng = Engine()
    for f, v in g["inserts"]:
        eng.add(f, v)
    for topic, want in g["matches"]:
        assert eng.matches(topic) == sorted(want), topic


def test_tokenizer_matches_host_dictionary():
    eng = Engine()
    filters = ["a/b/c", "$SYS/x", "/lead", "trail/", "x" * 27 + "/" + "y" * 28 + "/" + "z" * 300, "dev-0000001/+/#"]
    for i, f in enumerate(filters):
        eng.add(f, i)
    topics = ["a/b/c", "a//c", "$SYS/x", "x/$SYS", "a/b+", "a/#/c", "a/#", "+", "", "/", "x" * 27, "y" * 28, "z" * 300,
              "z" * 299, "nope", "a/b/c/" + "/".join(["q"] * 40)]
    toks, meta = eng.tokenize(topics, max_tok=8)
    inv = (meta >> 31) & 1
    assert inv.tolist() == [0, 0, 0, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0]
    nlev = meta & 0xFFFFFF
    assert nlev[0] == 3 and nlev[1] == 3 and nlev[8] == 1 and nlev[9] == 2 and nlev[15] == 43
    assert (meta[2] >> 30) & 1 == 1 and (meta[0] >> 30) & 1 == 0
    a, b, c = toks[0, 0], toks[1, 0], toks[2, 0]
    assert a >= 4 and b >= 4 and c >= 4 and len({a, b, c}) == 3
    assert toks[1, 1] == 3                       # Blank
    assert toks[0, 6] == a and toks[1, 6] == 2   # "a/#"
    assert toks[0, 7] == 1                       # "+"
    assert toks[0, 8] == 3 and toks[0, 9] == 3 and toks[1, 9] == 3
    assert toks[0, 10] >= 4 and toks[0, 11] >= 4 and toks[0, 12] >= 4   # 27 / 28 / 300-byte levels are in the dictionary
    assert toks[0, 13] == 0 and toks[0, 14] == 0                         # unknown strings


def test_c1_bit_exact_every_topic():
    cfg = wl.C1
    sb, so, sv = wl.gen_subs(cfg)
    tb, to = wl.gen_topics(cfg)
    eng, tree = Engine(), orc.TopicTree()
    assert eng.bulk_load(sb, so, sv) == tree.bulk_insert(sb, so, sv)
    res = eng.match_batch(tb, to)
    want = tree.match_batch(tb, to)
    _assert_same(res, want)
    assert res.needed == int(want["counts"].clip(0).sum())


@pytest.mark.parametrize("seed,tiny_windows", [(11, False), (12, False), (13, False), (14, True), (15, True)])
def test_random_differential_with_mutations(seed, tiny_windows, monkeypatch):
    if tiny_windows:      # 8-slot windows of the edge table: windows double, the table re-hashes, '+' slots move between flushes
        monkeypatch.setenv("GM_WIN_MIN_SLOTS_LOG2", "3")
    rng = random.Random(seed)
    eng, tree = Engine(), orc.TopicTree()
    live = []
    for rnd in range(6):
        for _ in range(400):
            if live and rng.random() < 0.3:
                f, v = rng.choice(live)
                try:
                    got = eng.remove(f, v)
                except GpuMqttError:
                    continue
                assert got == tree.remove(f, v)
            else:
                f, v = rand_filter(rng), rng.choice([0, 1, 2, 3, 2**31 + 5, 2**32 - 1, rng.randint(0, 60)])
                try:
                    got = eng.add(f, v)
                except GpuMqttError as ex:
                    assert ex.code == N.GM_ERR_INVALID_TOPIC
                    continue
                assert got == tree.insert(f, v)
                live.append((f, v))
        topics = [rand_topic(rng, max_depth=12) for _ in range(1500)]
        tb, to = pack(topics)
        res = eng.match_batch(tb, to)       # implicit flush: sees every mutation above
        want = tree.match_batch(tb, to)
        _assert_same(res, want)
        st = eng.stats()
        assert st["values"] == tree.values_size() and st["nodes"] == tree.nodes_size()


def test_c2_scaled_parity_and_work_counters():
    cfg = wl.C2.scaled(n_subs=200_000, n_topics=50_000)
    sb, so, sv = wl.gen_subs(cfg)
    tb, to = wl.gen_topics(cfg)
    eng, tree = Engine(filters_hint=cfg.n_subs), orc.TopicTree()
    assert eng.bulk_load(sb, so, sv) == tree.bulk_insert(sb, so, sv, nthreads=4)
    res = eng.match_batch(tb, to)
    want = tree.match_batch(tb, to, nthreads=4)
    _assert_same(res, want)
    # device-resident entry point + exact work counters == the oracle's (no removals: no dead nodes; the Bloom
    # mask only skips probes that would miss, which the oracle counts in E as well -> compare V,F,M,L,B)
    dev = torch.device("cuda")
    d_blob = torch.from_numpy(tb).to(dev)
    d_offs = torch.from_numpy(to.view(np.int32)).to(dev)
    n = len(to) - 1
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device=dev)
    d_ids = torch.zeros(max(1, res.needed), dtype=torch.int32, device=dev)
    d_needed = torch.zeros(1, dtype=torch.int64, device=dev)
    d_status = torch.zeros(n, dtype=torch.int32, device=dev)
    work = eng.match_batch_device(d_blob, d_offs, d_spans, d_ids, d_needed, d_status, torch.cuda.current_stream().cuda_stream, work=True)
    torch.cuda.synchronize()
    c = want["counters"]
    assert int(d_needed.item()) == res.needed == c["M"]
    assert (work["visited"], work["filters"], work["ids"], work["levels"], work["bytes"]) == (c["V"], c["F"], c["M"], c["L"], c["B"])
    assert work["probed"] == c["E"]
    from rmqtt_b200.engine import MatchResult
    res2 = MatchResult(d_spans.cpu().numpy().view(np.uint32), d_ids.cpu().numpy().view(np.uint32), d_status.cpu().numpy(), res.needed)
    _assert_same(res2, want)


def test_capacity_protocol_and_invalid_topics():
    eng = Engine()
    for i in range(100):
        eng.add("a/+", i)
    tb, to = pack(["a/b", "a/b+", "a/c", "$x/#/y", "zzz"])
    with pytest.raises(GpuMqttError) as ei:
        eng.match_batch(tb, to, cap_ids=150)
    assert ei.value.code == N.GM_ERR_CAPACITY
    res = eng.match_batch(tb, to)
    assert res.needed == 200
    assert res.status.tolist() == [0, N.GM_ERR_INVALID_TOPIC, 0, N.GM_ERR_INVALID_TOPIC, 0]
    assert res.sorted_list(0) == list(range(100)) and res.sorted_list(1) is None and res.sorted_list(4) == []


def test_deep_topics_and_heavy_hitters_take_the_deferred_path():
    eng, tree = Engine(), orc.TopicTree()
    deep = "/".join(f"l{i}" for i in range(20))
    fl = [deep, "/".join(["+"] * 20), "l0/l1/#", deep + "/#", "/".join(["l0"] + ["+"] * 10) + "/#"]
    for i, f in enumerate(fl):
        assert eng.add(f, i) == tree.insert(f, i)
    for v in range(5000):
        eng.add("hot/+", v); tree.insert("hot/+", v)
    topics = [deep, deep + "/x", "l0/l1", "hot/a", "hot", "l0/" + "/".join(["q"] * 19)] * 50
    tb, to = pack(topics)
    _assert_same(eng.match_batch(tb, to), tree.match_batch(tb, to))


def test_manual_flush_fence():
    eng = Engine(manual_flush=True)
    eng.add("a/b", 1)
    eng.flush()
    assert eng.matches("a/b") == [1]
    eng.add("a/b", 2)
    assert eng.matches("a/b") == [1]          # staged, not yet visible
    eng.flush()
    assert eng.matches("a/b") == [1, 2]
    eng.remove("a/b", 1)
    eng.flush()
    assert eng.matches("a/b") == [2]


def test_manual_flush_snapshot_survives_table_growth():
    """With GM_FLAG_MANUAL_FLUSH the kernels must keep seeing the tables as of the last flush, even when the host
    mirror has meanwhile re-hashed its edge table / dictionary (new geometry, new window count, deeper filters)."""
    rng = random.Random(3)
    eng, old, new = Engine(manual_flush=True), orc.TopicTree(), orc.TopicTree()
    for i in range(60):
        f = f"r{i % 5}/s{i % 7}/+/x{i}"
        eng.add(f, i); old.insert(f, i); new.insert(f, i)
    eng.flush()
    before = eng.stats()
    for i in range(6000):                       # grows edges (1 K slots -> >16 K), the dictionary and max_depth; nothing shipped
        f = f"r{i % 5}/s{i % 7}/d{i}/x{i % 60}/deep/er/than/before" if i % 3 else f"+/s{i % 7}/n{i}"
        eng.add(f, 1000 + i); new.insert(f, 1000 + i)
    assert eng.stats()["edge_slots"] > before["edge_slots"]
    topics = [f"r{rng.randrange(5)}/s{rng.randrange(7)}/d{rng.randrange(6000)}/x{rng.randrange(60)}" for _ in range(2000)]
    topics += [f"q/s{rng.randrange(7)}/n{rng.randrange(6000)}" for _ in range(500)]
    tb, to = pack(topics)
    _assert_same(eng.match_batch(tb, to), old.match_batch(tb, to))       # staged, not visible
    eng.flush()
    _assert_same(eng.match_batch(tb, to), new.match_batch(tb, to))


def test_acl_rule_tree_shape():
    """SURVEY §8(f) rank 2 — other TopicTree<V> users ride the same ABI: an ACL rule set is a small tree of topic
    filters (rmqtt-plugins/rmqtt-acl/src/config.rs:291-326) asked `is_match(topic)` on every PUBLISH / SUBSCRIBE;
    one engine per rule tree, is_match == "the match list is non-empty" (trie.rs:138-140)."""
    rng = random.Random(9)
    allow, deny, o_allow, o_deny = Engine(), Engine(), orc.TopicTree(), orc.TopicTree()
    for i in range(200):
        f = rand_filter(rng, 4)
        eng, tree = (allow, o_allow) if i % 3 else (deny, o_deny)
        try:
            eng.add(f, i)
        except GpuMqttError:
            continue
        tree.insert(f, i)
    topics = [rand_topic(rng, 5) for _ in range(4000)]
    tb, to = pack(topics)
    for eng, tree in ((allow, o_allow), (deny, o_deny)):
        got = eng.match_batch(tb, to).counts()
        want = tree.match_batch(tb, to, want_ids=False)["counts"]
        assert ((got > 0) == (want > 0)).all() and (got == want).all()


def test_extra_trees_ride_in_the_same_batch():
    """SURVEY §8(f) rank 2 as the survey words it: the ACL allow / deny rule trees are EXTRA ROOTS of the same engine
    (gm_sub_add_tree) and a PUBLISH's subscription match and its two ACL checks are three rows of ONE batch
    (gm_match_batch_trees) — one set of launches, not one engine and five launches per tree."""
    rng = random.Random(19)
    eng = Engine()
    trees = {0: orc.TopicTree(), 1: orc.TopicTree(), 2: orc.TopicTree(), 7: orc.TopicTree()}
    v = 0
    for _ in range(900):
        f = rand_filter(rng, 4)
        tr = rng.choice([0, 0, 1, 2, 7])
        v += 1
        try:
            ch = eng.add_tree(tr, f, v) if tr else eng.add(f, v)
        except GpuMqttError:
            continue
        assert ch == trees[tr].insert(f, v)
    for tr in (1, 2):                                   # root wildcards of an extra tree obey the `$`-rule at THEIR root
        for f in ("#", "+/x", "$SYS/#"):
            v += 1
            assert eng.add_tree(tr, f, v) == trees[tr].insert(f, v)
    topics = [rand_topic(rng, 5) for _ in range(1500)] + ["$SYS/x", "$SYS", "a/x", "x"]

    def check():
        rows, row_tree = [], []
        for t in topics:
            for tr in (0, 1, 2, 7, 9):                  # 9: a tree that does not exist -> empty list
                rows.append(t); row_tree.append(tr)
        tb, to = pack(rows)
        res = eng.match_batch_trees(tb, to, np.asarray(row_tree, dtype=np.uint32))
        for i, (t, tr) in enumerate(zip(rows, row_tree)):
            want = trees[tr].matches(t) if tr in trees else ([] if trees[0].matches(t) is not None else None)   # an invalid topic is an Err for any tree
            assert res.sorted_list(i) == (sorted(want) if want is not None else None), (t, tr)
        # tree 0 through the ordinary entry point is unaffected by its neighbours
        tb0, to0 = pack(topics)
        _assert_same(eng.match_batch(tb0, to0), trees[0].match_batch(tb0, to0))

    check()
    for f, val in (("#", 100001), ("+/x", 100002)):     # mutate an extra tree, flush, re-check; then compact (trees survive)
        assert eng.add_tree(7, f, val) == trees[7].insert(f, val)
    assert eng.remove_tree(1, "#", v - 5) == trees[1].remove("#", v - 5)
    check()
    eng.compact()
    check()


def test_full_size_properties_c3_shape():
    """Size-independent properties at a large size (no oracle): match counts are invariant under batch order;
    adding a `#` subscriber raises every non-`$` topic's count by exactly one; removing it restores them."""
    cfg = wl.C3.scaled(n_subs=2_000_000, n_topics=300_000)
    sb, so, sv = wl.gen_subs(cfg)
    tb, to = wl.gen_topics(cfg)
    eng = Engine(filters_hint=cfg.n_subs)
    eng.bulk_load(sb, so, sv)
    r1 = eng.match_batch(tb, to)
    c1 = r1.counts()
    assert (c1 >= 0).all() and c1.sum() == r1.needed
    topics = wl.unpack(tb, to)
    perm = np.random.default_rng(5).permutation(len(topics))
    pb, po = pack([topics[i] for i in perm])
    r2 = eng.match_batch(pb, po)
    assert (r2.counts() == c1[perm]).all()
    k1, i1 = r1.canonical()
    k2, i2 = r2.canonical()
    inv = np.argsort(perm)
    st = np.zeros(len(c1) + 1, dtype=np.int64); np.cumsum(c1[perm], out=st[1:])
    # spot-check multisets of 2000 topics across the permutation
    s1 = np.zeros(len(c1) + 1, dtype=np.int64); np.cumsum(c1, out=s1[1:])
    for t in range(0, len(c1), max(1, len(c1) // 2000)):
        j = inv[t]
        assert (i1[s1[t]:s1[t + 1]] == i2[st[j]:st[j + 1]]).all()
    eng.add("#", 0xABCDEF)
    assert (eng.match_batch(tb, to).counts() == c1 + 1).all()
    eng.remove("#", 0xABCDEF)
    assert (eng.match_batch(tb, to).counts() == c1).all()


def test_empty_engine_empty_batch_and_blank_topics():
    eng = Engine()
    assert eng.matches("a/b") == []                      # no filters at all
    res = eng.match_topics([])
    assert len(res) == 0 and res.needed == 0
    eng.add("", 1)                                       # the empty filter is [Blank] (topic.rs:497)
    eng.add("/", 2)
    eng.add("+", 3)
    eng.add("#", 4)
    tree = orc.TopicTree()
    for f, v in (("", 1), ("/", 2), ("+", 3), ("#", 4)):
        tree.insert(f, v)
    topics = ["", "/", "//", "a", "$", "$/", "+", "#"]
    tb, to = pack(topics)
    _assert_same(eng.match_batch(tb, to), tree.match_batch(tb, to))


def test_capacity_error_reports_needed_across_pipeline_chunks():
    cfg = wl.C2.scaled(n_subs=50_000, n_topics=300_000)   # > 2 chunks of the pipelined host path
    sb, so, sv = wl.gen_subs(cfg)
    tb, to = wl.gen_topics(cfg)
    eng = Engine()
    eng.bulk_load(sb, so, sv)
    full = eng.match_batch(tb, to)
    assert full.needed == int(full.counts().sum()) > 1000
    with pytest.raises(GpuMqttError) as ei:
        eng.match_batch(tb, to, cap_ids=full.needed // 3)
    assert ei.value.code == N.GM_ERR_CAPACITY
    again = eng.match_batch(tb, to, cap_ids=full.needed)          # exactly enough
    assert (again.counts() == full.counts()).all()
    c1, i1 = full.canonical(); c2, i2 = again.canonical()
    assert (i1 == i2).all()


def test_compact_on_device_keeps_parity():
    rng = random.Random(77)
    eng, tree = Engine(), orc.TopicTree()
    rtree, rtopics = orc.RetainTree(), []
    for i in range(800):                      # the retained tree shares the dictionary that compaction re-labels
        t = rand_topic(rng, 6)
        try:
            eng.retain_set(t, i)
        except GpuMqttError:
            continue
        rtree.insert(t, i)
        rtopics.append(t)
    live = []
    for _ in range(3000):
        f, v = rand_filter(rng), rng.randint(0, 30)
        try:
            eng.add(f, v)
        except GpuMqttError:
            continue
        tree.insert(f, v)
        live.append((f, v))
    for f, v in live[:2000]:
        assert eng.remove(f, v) == tree.remove(f, v)
    topics = [rand_topic(rng, 9) for _ in range(3000)]
    tb, to = pack(topics)
    _assert_same(eng.match_batch(tb, to), tree.match_batch(tb, to))
    eng.compact()
    st = eng.stats()
    assert st["device_nodes"] == st["nodes"] == tree.nodes_size() and st["garbage_value_words"] == 0
    _assert_same(eng.match_batch(tb, to), tree.match_batch(tb, to))
    eng.add("q/+/r", 9); tree.insert("q/+/r", 9)
    assert eng.matches("q/x/r") == tree.matches("q/x/r")
    filters = [f for f in (rand_filter(rng) for _ in range(600)) if orc.topic_parse(f) is not None]
    fb, fo = pack(filters)
    _assert_same(eng.retain_match_batch(fb, fo), rtree.match_batch(fb, fo))


def test_tokenizer_fuzz_against_topic_from_str():
    """SWAR tokeniser vs the oracle's Topic::from_str on random byte soup: validity, level count, `$` flag."""
    rng = random.Random(2024)
    alphabet = [b"/", b"/", b"+", b"#", b"$", b"a", b"b", b"cd", b"\xc3\xa9", b"\x7f", b" ", b"0", b"xyz", b"-", b"\xf0\x9f\x98\x80"]
    topics = []
    for _ in range(20000):
        n = rng.randint(0, 14)
        topics.append(b"".join(rng.choice(alphabet) for _ in range(n)))
    topics += [b"a" * 26 + b"/x", b"a" * 27 + b"/x", b"a" * 28 + b"/x", b"a" * 29 + b"+", b"/" * 40, b"a/" * 30 + b"#", b"$" * 3]
    eng = Engine()
    for i, f in enumerate(["a/b", "cd/+", "$/#", "a" * 27, "a" * 28]):
        eng.add(f, i)
    toks, meta = eng.tokenize(topics, max_tok=8)
    for i, t in enumerate(topics):
        want = orc.topic_parse(t)
        inv = bool(meta[i] >> 31)
        assert inv == (want is None), t
        if want is not None:
            assert int(meta[i] & 0xFFFFFF) == len(t.split(b"/")), t
            assert bool((meta[i] >> 30) & 1) == (want[0] == "Metadata"), t
            for l, kind in enumerate(want[:8]):
                tk = int(toks[l, i])
                if kind == "Single":
                    assert tk == 1
                elif kind == "Multi":
                    assert tk == 2
                elif kind == "Blank":
                    assert tk == 3
                else:
                    assert tk == 0 or tk >= 4
