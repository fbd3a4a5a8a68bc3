"""What choosing shared-subscription members on the device saves: gmr_matches_batch (every member of every matched group is
returned) against gmr_matches_batch_shared (one member per group and appearance, chosen by k_relations_choose), on the same
router.

Workload: the C2 subscriptions scaled like bench.py's relations leg (100 K numbered subscriptions, 20 K-topic batch; --full for
C2's 1 M / 100 K), plus shared groups of 4, 64 and 1 024 members on wildcard filters that many topics match: `#`, and
`<level0>/#` for the most frequent first topic levels.  A third of the members are told they are offline.

Prints one JSON object: per entry point the relations returned per batch, gmr_last_timing's device / host ms and the call ms
(medians of --reps calls after one warm-up), with the GPU name and power limit read in the same run.
    python tools/bench_shared_choice.py [--full] [--reps 6]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from collections import Counter
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from rmqtt_b200 import _native as N          # noqa: E402
from rmqtt_b200 import workload as wl         # noqa: E402
from rmqtt_b200.router import GpuRouter, Id, SubscriptionOptions   # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power = [x.strip() for x in out.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as exc:                  # the numbers are still printed; say what could not be read
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({exc.__class__.__name__})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true")
    ap.add_argument("--reps", type=int, default=6)
    a = ap.parse_args()
    cfg = wl.C2 if a.full else wl.C2.scaled(n_subs=100_000, n_topics=20_000, name="C2-scaled")
    sb, so, sv = wl.gen_subs(cfg)
    tb, to = wl.gen_topics(cfg)
    n = cfg.n_topics
    r = GpuRouter()
    lib = N.lib()
    rng = np.random.default_rng(7)
    nodes = rng.integers(1, 4, size=len(sv)).astype(np.uint64)
    clients = (sv // 2).astype(np.uint32)
    flags = (rng.random(len(sv)) < 0.5).astype(np.uint8)
    flags = flags[clients % len(flags)] | ((rng.random(len(sv)) < 0.1).astype(np.uint8) << 1)
    sub_ids = np.where(flags & 1, 1 + (sv % 7), 0).astype(np.uint32)
    added = C.c_uint64(0)
    assert lib.gmr_add_batch_numbered(r._h, sb.ctypes.data, so.ctypes.data, len(sv), nodes.ctypes.data, clients.ctypes.data, flags.ctypes.data,
                                      sub_ids.ctypes.data, C.byref(added)) == 0
    # shared groups on wildcard filters the batch matches often
    topics = [bytes(tb[to[i]:to[i + 1]]).decode() for i in range(min(n, 5000))]
    level0 = [k for k, _ in Counter(t.split("/")[0] for t in topics).most_common(3)]
    filters = ["#"] + [f"{l0}/#" for l0 in level0]
    for fi, f in enumerate(filters):
        for size in (4, 64, 1024):
            name = f"g{size}"
            for k in range(size):
                ident = Id(1 + k % 3, f"share-{fi}-{size}-{k}", k)
                r.add(f, ident, SubscriptionOptions(qos=1, is_v5=k % 2 == 1, sub_id=k % 5, shared_group=name))
                if k % 3 == 0:
                    r.set_online(ident.node_id, ident.client_id, False)
    spans = np.zeros((n, 2), dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    cap_r, cap_s = 64 * n, 16 * n
    rels = (N.GmSubRelation * cap_r)()
    sids = np.zeros(cap_s, dtype=np.uint32)
    res = {}
    for label in ("gmr_matches_batch", "gmr_matches_batch_shared"):
        nr, ns = C.c_uint64(0), C.c_uint64(0)
        dev_ms, host_ms, wall = [], [], []
        k = 0
        while k < a.reps + 1:
            args = (None, tb.ctypes.data, to.ctypes.data, n, spans.ctypes.data, rels, cap_r, sids.ctypes.data, cap_s, C.byref(nr), C.byref(ns), status.ctypes.data)
            t0 = time.perf_counter()
            rc = lib.gmr_matches_batch(r._h, *args) if label == "gmr_matches_batch" else lib.gmr_matches_batch_shared(r._h, 1000 + k, *args)
            wall.append((time.perf_counter() - t0) * 1e3)
            if rc == N.GM_ERR_CAPACITY:                      # grow the outputs, and time the call again
                cap_r, cap_s = max(cap_r, int(nr.value)), max(cap_s, int(ns.value), 1)
                rels = (N.GmSubRelation * cap_r)()
                sids = np.zeros(cap_s, dtype=np.uint32)
                wall.pop()
                continue
            assert rc == 0, (label, rc, nr.value, ns.value)
            k += 1
            d, h = C.c_double(0), C.c_double(0)
            lib.gmr_last_timing(r._h, C.byref(d), C.byref(h))
            dev_ms.append(d.value)
            host_ms.append(h.value)
        assert len(wall) == a.reps + 1
        res[label] = {"relations_per_batch": int(nr.value), "sub_ids_per_batch": int(ns.value), "device_ms": float(np.median(dev_ms[1:])),
                      "host_ms": float(np.median(host_ms[1:])), "call_ms": float(np.median(wall[1:]))}
    print(json.dumps({"workload": f"{cfg.name}: {int(added.value)} numbered subscriptions + shared groups of 4, 64 and 1024 members on "
                                  f"{filters}, a third of the members offline; {n}-topic batch, host buffers",
                      **gpu_info(), **res}, indent=1))


if __name__ == "__main__":
    main()
