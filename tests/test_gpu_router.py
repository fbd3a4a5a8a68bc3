"""GPU tier: the C++ GpuRouter (DefaultRouter semantics above the engine) against the oracle's restatement of
rmqtt/src/router.rs:162-248, 417-479 and rmqtt/src/types.rs:470-508."""
import random

import pytest

from oracle import oracle as orc
from rmqtt_b200.engine import GpuMqttError
from rmqtt_b200 import _native as N
from rmqtt_b200.router import GpuRouter, Id, SubscriptionOptions

from _gen import rand_filter, rand_topic

pytestmark = pytest.mark.gpu


def test_add_remove_counters_and_id_rule():
    r, o = GpuRouter(), orc.Router()
    a, b = Id(1, "c1", 11), Id(1, "c2", 22)
    r.add("a/+", a); o.add_full("a/+", "c1", 0, 11, 1)
    r.add("a/+", b); o.add_full("a/+", "c2", 1, 22, 1)
    r.add("a/b", a); o.add_full("a/b", "c1", 2, 11, 1)
    with pytest.raises(GpuMqttError) as ei:
        r.add("a/#/b", a)
    assert ei.value.code == N.GM_ERR_INVALID_TOPIC
    assert (r.topics(), r.routes(), r.topics_tree()) == (o.topics(), o.routes(), 3) == (2, 3, 3)
    assert not r.remove("a/+", Id(1, "c1", 99))            # Id mismatch (router.rs:444-451)
    assert r.remove("a/+", a) and o.remove("a/+", "c1", 11) == 1
    assert r.remove("a/+", b) and o.remove("a/+", "c2", 22) == 1
    assert (r.topics(), r.routes()) == (o.topics(), o.routes()) == (1, 1)
    got = r.matches(Id(9, "pub"), "a/b")
    assert [(x.topic_filter, x.client_id) for x in got] == [("a/b", "c1")]
    r.add("a/b", Id(1, "c1", 11), SubscriptionOptions(qos=1))   # re-subscribe replaces, count unchanged (router.rs:430-433)
    assert r.routes() == 1
    assert r.matches(Id(9, "pub"), "a/b+") is None


@pytest.mark.parametrize("seed", [31, 32])
def test_random_differential_vs_oracle_router(seed):
    rng = random.Random(seed)
    r, o = GpuRouter(), orc.Router()
    subs = {}
    clients = [Id(rng.randint(1, 3), f"c{k}", 100 + k) for k in range(25)]
    v5flag = {}
    rel = 0
    for step in range(700):
        cid = rng.choice(clients)
        if subs and rng.random() < 0.25:
            (f, c) = rng.choice(list(subs))
            ident = subs[(f, c)]
            wrong = rng.random() < 0.2
            use = Id(ident.node_id, ident.client_id, 7) if wrong else ident
            got = r.remove(f, use)
            want = o.remove(f, ident.client_id, use.tag)
            assert got == (want == 1)
            if got:
                del subs[(f, c)]
        else:
            f = rand_filter(rng, 5)
            v5 = rng.random() < 0.5
            opts = SubscriptionOptions(qos=rng.randint(0, 2), is_v5=v5, no_local=v5 and rng.random() < 0.5,
                                       sub_id=rng.randint(1, 9) if v5 and rng.random() < 0.6 else 0,
                                       shared_group=rng.choice(["", "", "", "g1", "g2"]))
            rel += 1
            try:
                r.add(f, cid, opts)
            except GpuMqttError as ex:
                assert ex.code == N.GM_ERR_INVALID_TOPIC
                assert not o.add_full(f, cid.client_id, rel, cid.tag, cid.node_id, opts.is_v5, opts.no_local, opts.sub_id, opts.shared_group)
                continue
            assert o.add_full(f, cid.client_id, rel, cid.tag, cid.node_id, opts.is_v5, opts.no_local, opts.sub_id, opts.shared_group)
            subs[(f, cid.client_id)] = cid
            v5flag[(f, cid.client_id)] = v5
        if step % 100 == 99:
            assert (r.topics(), r.routes()) == (o.topics(), o.routes())
            topics = [rand_topic(rng, 6) for _ in range(300)]
            pubs = [rng.choice(clients) for _ in topics]
            got = r.matches_batch(topics, pubs)
            for t, p, g in zip(topics, pubs, got):
                want = o.matches_full(t, p.node_id, p.client_id, p.tag)
                if want is None:
                    assert g is None, t
                    continue
                lines, groups = [], {}
                for x in g:
                    if x.group:
                        groups.setdefault((x.group, x.topic_filter), []).append(f"{x.node_id}:{x.client_id}")
                    elif v5flag[(x.topic_filter, x.client_id)]:
                        lines.append(f"5|{x.node_id}|{x.client_id}|" + ",".join(str(s) for s in sorted(x.sub_ids)))
                    else:
                        lines.append(f"3|{x.node_id}|{x.topic_filter}|{x.client_id}")
                # shared groups: the oracle emits one line per matched-filter occurrence and group with all members
                wl = [w for w in want if not w.startswith("g|")]
                wg = sorted(w.split("|", 3)[3] for w in want if w.startswith("g|"))
                assert sorted(lines) == wl, t
                # members per (filter, group): an occurrence-multiset; compare flattened member multisets
                got_members = sorted(m for ms in groups.values() for m in ms)
                want_members = sorted(m for w in wg for m in w.split(";"))
                assert got_members == want_members, t


@pytest.mark.parametrize("n_clients,per_client", [(60, 3), (300, 2), (5, 40)])
def test_v5_per_client_dedup_on_the_device_and_its_host_fallback(n_clients, per_client):
    """types.rs:488-506 on the device (k_relations): a v5 client matching through several filters gets ONE relation with all
    its subscription identifiers; a topic with more v5 relations than the kernel stages (256) is finished on the host."""
    r, o = GpuRouter(), orc.Router()
    filters = ["t/+/x", "t/a/+", "t/#", "+/a/x", "t/a/x", "#", "t/+/+", "+/+/x", "+/a/+", "+/+/+"]
    filters += [f"t/a/x/{k}/#" for k in range(40)]           # do not match the probe topic
    filters = (filters[:10] * 4)[:per_client] if per_client <= 10 else [f"t/a/x" if k == 0 else (filters[k % 10] if k < 10 else f"q{k}/+/x") for k in range(per_client)]
    filters = list(dict.fromkeys(filters))                    # distinct filters per client
    rel = 0
    v5flag = {}
    for c in range(n_clients):
        cid = Id(1 + c % 2, f"c{c}", 500 + c)
        for j, f in enumerate(filters):
            rel += 1
            v5 = c % 5 != 0                                    # every fifth client is v3: no de-dup for it
            opts = SubscriptionOptions(qos=1, is_v5=v5, no_local=v5 and c % 7 == 0, sub_id=(1 + (c + j) % 9) if v5 and (c + j) % 3 else 0)
            r.add(f, cid, opts)
            assert o.add_full(f, cid.client_id, rel, cid.tag, cid.node_id, opts.is_v5, opts.no_local, opts.sub_id, "")
            v5flag[(f, cid.client_id)] = v5
    topics = ["t/a/x", "t/b/x", "z/a/x", "nomatch"]
    pubs = [Id(1, "c0", 500), Id(2, "c7", 507), Id(1, "c14", 514), Id(9, "nobody", 1)]      # c7 and c14 are v5 + no_local: dropped for their own PUBLISH
    got = r.matches_batch(topics, pubs)
    for t, p, g in zip(topics, pubs, got):
        want = o.matches_full(t, p.node_id, p.client_id, p.tag)
        lines = []
        for x in g:
            if v5flag[(x.topic_filter, x.client_id)]:
                lines.append(f"5|{x.node_id}|{x.client_id}|" + ",".join(str(s) for s in sorted(x.sub_ids)))
            else:
                lines.append(f"3|{x.node_id}|{x.topic_filter}|{x.client_id}")
        assert sorted(lines) == want, t


@pytest.mark.parametrize("shared", [False, True])
def test_merged_v5_record_carries_the_smallest_handle(shared):
    """A v5 client matched through several subscriptions gets the record of its smallest handle, from the device ("u/a/x": 10 v5
    relations) and from the host fallback ("t/a/x": 600, more than the kernel stages), in gmr_matches_batch and
    gmr_matches_batch_shared.  Every client subscribes to the filter the walk lists last first, so its first-listed handle is
    not its smallest."""
    r = GpuRouter()
    sizes = {"t": 300, "u": 5}
    for prefix, n_clients in sizes.items():
        for c in range(n_clients):
            for f in (f"{prefix}/a/x", f"{prefix}/#"):         # the walk lists "<prefix>/#" before "<prefix>/a/x"
                r.add(f, Id(1, f"{prefix}{c}", c), SubscriptionOptions(qos=1, is_v5=True, sub_id=1 + c % 7))
    handle = {r._relation(h): h for h in range(2 * sum(sizes.values()))}
    got = r.matches_batch(["t/a/x", "u/a/x"], seed=7 if shared else None)
    for (prefix, n_clients), rels in zip(sizes.items(), got):
        assert sorted(x.client_id for x in rels) == sorted(f"{prefix}{c}" for c in range(n_clients))
        for x in rels:
            c = int(x.client_id[1:])
            assert x.sub_ids == [1 + c % 7] * 2
            assert handle[(x.topic_filter, x.client_id)] == min(handle[(f, x.client_id)] for f in (f"{prefix}/a/x", f"{prefix}/#")), x


def test_secondary_readers_through_descriptor_mode():
    """_has_matches / _get_routes / Router::get (router.rs:139-158, 522-546) answered by the engine (descriptor mode: one
    descriptor per matched filter), against the oracle's restatement — no second CPU trie."""
    rng = random.Random(77)
    r, o = GpuRouter(), orc.Router()
    clients = [Id(rng.randint(1, 4), f"c{k}", 100 + k) for k in range(30)]
    rel = 0
    for _ in range(600):
        f = rand_filter(rng, 5)
        cid = rng.choice(clients)
        rel += 1
        try:
            r.add(f, cid)
        except GpuMqttError:
            continue
        assert o.add_full(f, cid.client_id, rel, cid.tag, cid.node_id, False, False, 0, "")
    topics = [rand_topic(rng, 6) for _ in range(400)] + ["+/a", "a/#", "bad/#/x", "$SYS/x"]
    for t in topics:
        want_has, want_routes, want_get = o.readers(t, 0), o.readers(t, 1), o.readers(t, 2)
        if want_has is None:
            assert r.has_matches(t) is None and r.get(t) is None, t
            continue
        assert r.has_matches(t) == (want_has == ["1"]), t
        assert [f for _, f in r.get_routes(t, 5)] == want_routes, t
        assert [f"{n}|{f}" for n, f in r.get(t)] == want_get, t
