"""GPU tier of the shared-subscription choice: gmr_matches_batch_shared against the router-level restatement of
tests/_shared_oracle.py (rmqtt/src/router.rs:162-248 with the seeded draw of include/gpumqtt.h), the distribution of the
draw, large groups, the capacity protocol, and gm_relations_choose_device on caller-built tables."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

import _shared_oracle as SO
import test_shared_choice_cpu as CPU
from rmqtt_b200 import _native as N
from rmqtt_b200.engine import Engine, pack
from rmqtt_b200.router import GpuRouter, Id, SubscriptionOptions

from _gen import rand_filter, rand_topic

pytestmark = pytest.mark.gpu

CHI2_P001 = {2: 13.816, 9: 27.877}          # chi-square bound at p = 0.001 for 2 and 9 degrees of freedom


class Pair:
    """The GPU router and the restatement, driven together; keeps what the canonical lines need."""

    def __init__(self, manual=False):
        self.eng = Engine(manual_flush=manual)
        self.r, self.o = GpuRouter(self.eng), SO.SharedRouter()
        self.opts = {}                                       # (filter, client) -> (Id, SubscriptionOptions)

    def add(self, f, ident: Id, opts=SubscriptionOptions()):
        try:
            self.r.add(f, ident, opts)
            ok = True
        except Exception:
            ok = False
        assert ok == self.o.add(f, ident.node_id, ident.client_id, ident.tag, opts.is_v5, opts.no_local, opts.sub_id, opts.shared_group)
        if ok:
            self.opts[(f, ident.client_id)] = (ident, opts)

    def remove(self, f, ident: Id):
        got = self.r.remove(f, ident)
        assert got == self.o.remove(f, ident.node_id, ident.client_id, ident.tag)
        if got:
            del self.opts[(f, ident.client_id)]

    def set_online(self, ident: Id, on: bool):
        self.r.set_online(ident.node_id, ident.client_id, on)
        self.o.set_online(ident.node_id, ident.client_id, on)

    def canon(self, rels):
        if rels is None:
            return None
        lines = []
        for x in rels:
            ident, opts = self.opts[(x.topic_filter, x.client_id)]
            if opts.is_v5:
                lines.append(f"5|{x.node_id}|{x.client_id}|" + ",".join(str(i) for i in sorted(x.sub_ids)))
            elif x.group:
                name = self.r.group_members(x.group)[1]
                lines.append(f"s|{x.node_id}|{x.topic_filter}|{name}|{x.client_id}|{int(x.online)}")
            else:
                lines.append(f"3|{x.node_id}|{x.topic_filter}|{x.client_id}")
        return sorted(lines)

    def check(self, topics, pubs, seed):
        got = self.r.matches_batch_shared(topics, pubs, seed=seed)
        for row, (t, p) in enumerate(zip(topics, pubs)):
            want = self.o.matches(t, row, seed, (p.node_id, p.client_id, p.tag))
            assert self.canon(got[row]) == want, (t, row, seed)
        return got


@pytest.mark.parametrize("manual", [False, True])
def test_random_differential_vs_restatement(manual):
    rng = random.Random(41 + manual)
    P = Pair(manual)
    clients = [Id(rng.randint(1, 3), f"c{k}", 100 + k) for k in range(30)]
    filters = [rand_filter(rng, 4) for _ in range(25)] + ["t/#", "t/+", "+/+", "#"]
    groups = ["", "", "g1", "g2", "g3"]
    if manual:                                               # unshared relations first, made visible by an explicit flush
        for _ in range(80):
            c = rng.choice(clients)
            P.add(rng.choice(filters), c, SubscriptionOptions(is_v5=rng.random() < 0.5, no_local=rng.random() < 0.3, sub_id=rng.choice([0, 3, 5])))
        P.eng.flush()
    for step in range(25):
        for _ in range(rng.randint(5, 40)):
            c = rng.choice(clients)
            x = rng.random()
            if x < 0.15 and P.opts:
                f, cl = rng.choice(list(P.opts))
                g = P.opts[(f, cl)][0]
                if manual and not P.opts[(f, cl)][1].shared_group:
                    continue
                P.remove(f, g)
            elif x < 0.3:
                P.set_online(c, rng.random() < 0.5)
            else:
                f = rng.choice(filters)
                grp = rng.choice(groups[2:] if manual else groups)
                if manual and (f, c.client_id) in P.opts and not P.opts[(f, c.client_id)][1].shared_group:
                    continue                                 # keep every unshared relation as flushed
                opts = SubscriptionOptions(qos=1, is_v5=rng.random() < 0.5, no_local=rng.random() < 0.3, sub_id=rng.choice([0, 3, 5, 9]), shared_group=grp)
                P.add(f, c, opts)                            # a re-subscribe may change or drop the group
        topics = [rand_topic(rng, 4) for _ in range(40)] + ["t/+", "t/a", "a/b", "t/+/x"]
        pubs = [rng.choice(clients) for _ in topics]
        P.check(topics, pubs, rng.getrandbits(64))


def _chi2(counts):
    n = sum(counts)
    e = n / len(counts)
    return sum((c - e) ** 2 / e for c in counts)


def test_distribution_of_the_draw():
    P = Pair()
    members = [Id(1, f"m{k}", k) for k in range(10)]
    for m in members:
        P.add("t/#", m, SubscriptionOptions(shared_group="w"))
    topics = [f"t/x{i}" for i in range(20_000)]
    pub = [Id(9, "pub")] * len(topics)

    def draw(seed):
        got = P.r.matches_batch_shared(topics, pub, seed=seed)
        assert all(len(g) == 1 for g in got)
        return [g[0] for g in got]

    got = draw(2024)
    cnt = [sum(1 for g in got if g.client_id == m.client_id) for m in members]
    assert all(g.online for g in got) and _chi2(cnt) < CHI2_P001[9], cnt
    for m in members[3:]:
        P.set_online(m, False)
    got = draw(2025)
    cnt = [sum(1 for g in got if g.client_id == m.client_id) for m in members[:3]]
    assert sum(cnt) == len(topics) and all(g.online for g in got) and _chi2(cnt) < CHI2_P001[2], cnt
    for m in members[:3]:
        P.set_online(m, False)
    got = draw(2026)
    cnt = [sum(1 for g in got if g.client_id == m.client_id) for m in members]
    assert not any(g.online for g in got) and _chi2(cnt) < CHI2_P001[9], cnt
    # a group whose only member is the publisher, with no_local: nothing is chosen
    me = Id(5, "me", 1)
    P.add("solo/#", me, SubscriptionOptions(is_v5=True, no_local=True, shared_group="s"))
    assert P.r.matches_batch_shared(["solo/a"], [me], seed=1) == [[]]
    assert len(P.r.matches_batch_shared(["solo/a"], [Id(5, "me", 2)], seed=1)[0]) == 1


def test_large_group_among_many_small_ones():
    rng = random.Random(5)
    P = Pair()
    for k in range(5000):                                    # v3 members: no per-client merging, one record per choice
        P.add("big/#", Id(1 + k % 4, f"b{k}", k), SubscriptionOptions(shared_group="big"))
    for g in range(300):
        for k in range(rng.randint(1, 6)):
            P.add(f"big/{g % 10}/#" if g % 2 else "big/+/x", Id(2, f"s{g}_{k}", k), SubscriptionOptions(shared_group=f"sg{g}"))
    for k in range(0, 5000, 7):
        P.set_online(Id(1 + k % 4, f"b{k}"), False)
    topics = [f"big/{i % 10}/x" for i in range(24)] + ["big/+/x", "big/q"]
    pubs = [Id(1, "b0", 0)] * len(topics)
    got = P.check(topics, pubs, 77)
    plain = P.r.matches_batch(topics, pubs)
    for row, t in enumerate(topics):
        # exactly one record per (group, appearance): every matched group has an eligible member here
        vals = P.o.tree.matches(t)
        appearances = sum(len({r[5] for r in P.o.rel[P.o.filters[fi]].values()}) for fi in vals)
        assert len(got[row]) == appearances, (t, len(got[row]), appearances)
        members = sum(len(P.o.rel[P.o.filters[fi]]) for fi in vals)
        assert len(plain[row]) == members                    # gmr_matches_batch still returns every member
    assert sum(map(len, got)) * 30 < sum(map(len, plain))   # 4 286 chosen records against 144 399 members


def test_literal_plus_topic_gets_two_choices():
    P = Pair()
    for k in range(50):
        P.add("t/+", Id(1, f"m{k}", k), SubscriptionOptions(shared_group="g"))
    for seed in range(20):
        got = P.check(["t/+", "t/a"], [Id(9, "p")] * 2, seed)
        assert len(got[0]) == 2 and len(got[1]) == 1


def _plain_want(P, topic, pub):
    """gmr_matches_batch restated on the same relations: every shared member passes through as a line of its own."""
    lines, v5 = [], {}
    for fi in P.o.tree.matches(topic):
        filt = P.o.filters[fi]
        for client, (node, tag, is_v5, no_local, sub_id, group) in P.o.rel.get(filt, {}).items():
            if is_v5 and no_local and (pub.node_id, pub.client_id, pub.tag) == (node, client, tag):
                continue
            if group:
                lines.append(f"g|{node}|{filt}|{group}|{client}")
            elif is_v5:
                v5.setdefault((node, client), []).extend([sub_id] if sub_id else [])
            else:
                lines.append(f"3|{node}|{filt}|{client}")
    lines += [f"5|{node}|{client}|" + ",".join(map(str, sorted(ids))) for (node, client), ids in v5.items()]
    return sorted(lines)


def _plain_lines(P, rels):
    lines = []
    for x in rels:
        if x.group:
            assert not x.sub_ids
            lines.append(f"g|{x.node_id}|{x.topic_filter}|{P.r.group_members(x.group)[1]}|{x.client_id}")
        elif P.opts[(x.topic_filter, x.client_id)][1].is_v5:
            lines.append(f"5|{x.node_id}|{x.client_id}|" + ",".join(map(str, sorted(x.sub_ids))))
        else:
            lines.append(f"3|{x.node_id}|{x.topic_filter}|{x.client_id}")
    return sorted(lines)


def test_flagged_topics_finished_on_the_host():
    """Topics with more v5 relations than the kernel stages (256) are de-duplicated on the host: chosen v5 members (many of them
    clients with a plain v5 relation too), v3 group members, no_local drops and plain v5 relations, against the restatement.
    gmr_matches_batch on the same topics passes every member through, unmerged."""
    rng = random.Random(13)
    P = Pair()
    for k in range(300):                                     # 300 plain v5 relations on every "h/..." topic
        P.add("h/#", Id(1 + k % 2, f"p{k}", k), SubscriptionOptions(qos=1, is_v5=True, no_local=k % 5 == 0, sub_id=rng.choice([0, 3, 5, 9])))
    for k in range(0, 300, 3):                               # v5 members; the even ones are plain v5 clients as well
        P.add("h/+/x", Id(1 + k % 2, f"p{k}" if k % 2 == 0 else f"m{k}", k),
              SubscriptionOptions(qos=1, is_v5=True, no_local=k % 4 == 0, sub_id=rng.choice([0, 4, 7]), shared_group=f"v{k % 4}"))
    for k in range(40):
        P.add("h/a/+", Id(2, f"s{k}", k), SubscriptionOptions(shared_group=f"w{k % 3}"))
    for k in range(20):
        P.add("h/+/+", Id(1, f"d{k}", k))
    for k in range(0, 300, 7):
        P.set_online(Id(1 + k % 2, f"p{k}"), False)
    topics = ["h/a/x", "h/b/x", "h/a/y", "h/+/x", "q/a"]
    pubs = [Id(1, "p0", 0), Id(1, "p12", 12), Id(2, "s1", 1), Id(9, "nobody"), Id(1, "p20", 20)]
    for seed in range(6):
        P.check(topics, pubs, seed)
    plain = P.r.matches_batch(topics, pubs)
    for row, (t, p) in enumerate(zip(topics, pubs)):
        assert _plain_lines(P, plain[row]) == _plain_want(P, t, p), t


def _raw_shared(P, topics, seed, cap_rels, cap_subs=1 << 16):
    blob, offs = pack(topics)
    n = len(topics)
    spans = np.zeros((n, 2), dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    rels = (N.GmSubRelation * max(cap_rels, 1))()
    sids = np.zeros(cap_subs, dtype=np.uint32)
    nr, ns = C.c_uint64(0), C.c_uint64(0)
    rc = N.lib().gmr_matches_batch_shared(P.r._h, seed, None, blob.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p), n,
                                          spans.ctypes.data_as(C.c_void_p), rels, cap_rels, sids.ctypes.data_as(C.c_void_p), cap_subs,
                                          C.byref(nr), C.byref(ns), status.ctypes.data_as(C.c_void_p))
    return rc, int(nr.value), [(rels[k].handle, rels[k].group) for k in range(int(nr.value))] if rc == 0 else None


def test_capacity_protocol():
    P = Pair()
    for k in range(40):
        P.add("c/#", Id(1, f"m{k}", k), SubscriptionOptions(shared_group=f"g{k % 4}"))
        P.add("c/+", Id(1, f"d{k}", k))
    topics = [f"c/{i}" for i in range(30)]
    rc, need, _ = _raw_shared(P, topics, 3, 1 << 12)
    assert rc == 0 and need == 30 * (4 + 40)
    rc, n2, recs = _raw_shared(P, topics, 3, need)
    assert rc == 0 and n2 == need and len(recs) == need
    rc, n3, _ = _raw_shared(P, topics, 3, need - 1)
    assert rc == N.GM_ERR_CAPACITY and n3 == need


def test_choose_device_with_caller_tables():
    """gm_relations_choose_device on the synthetic corpus of the CPU tier, d_online = NULL, against the same Python model."""
    case = CPU.Case(seed=21)
    lists = case.lists()
    seed = 99
    n = len(lists)
    dev = torch.device("cuda")
    spans = np.zeros((n, 2), dtype=np.uint32)
    o = 0
    for i, l in enumerate(lists):
        spans[i] = (o, len(l))
        o += len(l)
    ids = np.asarray([h for l in lists for h in l] + [0], dtype=np.uint32)
    table = np.zeros((len(case.rels), 6), dtype=np.uint32)
    for h, r in enumerate(case.rels):
        table[h] = (r["node_id"], 0, r["client_key"], r["id_idx"], r["sub_id"], r["flags"])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).to(dev)   # noqa: E731
    d_spans, d_ids, d_pubs, d_rels = t(spans), t(ids), t(np.asarray(case.pubs, dtype=np.uint32)), t(table)
    d_groups, d_members = t(np.asarray(case.groups, dtype=np.uint32)), t(np.asarray(case.members, dtype=np.uint32))
    cap = len(ids) + 8
    d_ospans = torch.zeros(2 * n, dtype=torch.int32, device=dev)
    d_orels = torch.zeros(cap * 6, dtype=torch.int32, device=dev)
    d_subs = torch.zeros(cap, dtype=torch.int32, device=dev)
    d_needed = torch.zeros(3, dtype=torch.int64, device=dev)
    d_status = torch.zeros(n, dtype=torch.int32, device=dev)
    eng = Engine()

    class GmRelOut(C.Structure):
        _fields_ = [("d_spans", C.c_void_p), ("d_rels", C.c_void_p), ("cap_rels", C.c_uint64), ("d_sub_ids", C.c_void_p), ("cap_sub_ids", C.c_uint64),
                    ("d_needed", C.c_void_p), ("d_status", C.c_void_p)]

    out = GmRelOut(d_ospans.data_ptr(), d_orels.data_ptr(), cap, d_subs.data_ptr(), cap, d_needed.data_ptr(), d_status.data_ptr())
    g = N.GmRelGroups(d_groups.data_ptr(), case.n_groups, d_members.data_ptr(), None, 0, seed)
    stream = torch.cuda.current_stream()
    before = N.lib().gm_kernel_launches(eng._h)
    rc = N.lib().gm_relations_choose_device(eng._h, d_spans.data_ptr(), d_ids.data_ptr(), n, d_pubs.data_ptr(), d_rels.data_ptr(), len(case.rels),
                                            C.byref(g), C.byref(out), C.c_void_p(stream.cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    assert N.lib().gm_kernel_launches(eng._h) == before + 1
    o_spans = d_ospans.cpu().numpy().view(np.uint32).reshape(n, 2)
    o_rels = d_orels.cpu().numpy().view(np.uint32).reshape(cap, 6)
    o_subs = d_subs.cpu().numpy().view(np.uint32)
    status = d_status.cpu().numpy()
    want = CPU.model(case, lists, seed, None)
    for row in range(n):
        off, cnt = o_spans[row]
        got = []
        for k in range(off, off + cnt):
            r = o_rels[k]
            got.append((int(r[0]) | int(r[1]) << 32, int(r[2]), int(r[3]), tuple(sorted(int(x) for x in o_subs[r[4]:r[4] + r[5]]))))
        assert (sorted(got), int(status[row])) == want[row], row
    assert int(d_needed[0]) == sum(len(w[0]) for w in want)
