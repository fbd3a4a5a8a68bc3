import os, random, sys
from pathlib import Path
_ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(_ROOT)); sys.path.insert(0, str(_ROOT / "tests"))
os.environ["GM_WIN_MIN_SLOTS_LOG2"] = "3"
from oracle import oracle as orc
from rmqtt_b200.engine import Engine, GpuMqttError, pack
from _gen import rand_filter, rand_topic
rng = random.Random(5)
eng, tree, rt = Engine(), orc.TopicTree(), orc.RetainTree()
live, topics = [], []
for rnd in range(4):
    for _ in range(250):
        f, v = rand_filter(rng), rng.randint(0, 30)
        try:
            eng.add(f, v)
        except GpuMqttError:
            continue
        tree.insert(f, v); live.append((f, v))
    for f, v in live[::5]:
        assert eng.remove(f, v) == tree.remove(f, v)
    for _ in range(150):
        t = rand_topic(rng, 6)
        if orc.topic_parse(t) is None or "#" in t.split("/") or "+" in t.split("/"):
            continue
        assert eng.retain_set(t, len(topics)) == rt.remove(t); rt.insert(t, len(topics)); topics.append(t)
    for t in topics[::7]:
        assert eng.retain_remove(t) == rt.remove(t)
    ts = [rand_topic(rng, 12) for _ in range(600)]
    tb, to = pack(ts)
    res = eng.match_batch(tb, to)
    for i, t in enumerate(ts):
        assert res.sorted_list(i) == tree.matches(t), t
    c1, i1 = res.canonical()
    c2, i2 = eng.match_batch_via_desc(tb, to).canonical()            # descriptor mode (small-batch graph)
    assert (c1 == c2).all() and (i1 == i2).all()
    big = ts * 5                                                      # 3000 topics: the pipelined (chunked) path
    bb, bo = pack(big)
    rb = eng.match_batch(bb, bo)
    for i in range(0, len(big), 97):
        assert rb.sorted_list(i) == tree.matches(big[i])
    fs = [f for f in (rand_filter(rng, 6) for _ in range(300)) if orc.topic_parse(f) is not None]
    fb, fo = pack(fs)
    rr = eng.retain_match_batch(fb, fo)
    for i, f in enumerate(fs):
        assert rr.sorted_list(i) == rt.matches(f), f
    if rnd == 2:
        eng.compact()
print("memcheck workload ok", eng.debug_tables()["rstats"].tolist())
