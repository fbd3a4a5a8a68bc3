#!/usr/bin/env python
"""Single-SUBSCRIBE retained lookups on config C4 (5 M retained topics, filters from gen_retain_filters), one JSON line:

  * lone lookups: gm_retain_match_batch with n = 1, one filter after another from one thread, with the small-batch graphs on
    and off (debug_knob small_graphs) — p50 / p99 latency and lookups/s;
  * the retained batcher: gm_retain_batcher_probe at bursts 1, 64 and 2048 (closed loop);
  * optionally bench.py's C4 leg (--c4-leg), imported from bench.py, not changed;
  * the card's name and power limit, read in the same run.

Every lone lookup's handle multiset is checked against the same filter's list from one 100 K-filter batch.

--lib PATH runs against another build of libgpumqtt.so (an A/B comparison with an older build): entry points that build does
not export are reported as not measured.  Usage: python tools/bench_retain_batcher.py [--lib PATH] [--lone N] [--c4-leg] [--small]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:                  # noqa: BLE001
        return {"error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="another build of libgpumqtt.so")
    ap.add_argument("--lone", type=int, default=3000, help="lone lookups per graphs setting")
    ap.add_argument("--rounds", type=int, default=0, help="probe rounds per burst (0: about 3000 lookups per burst, at least 20 rounds)")
    ap.add_argument("--c4-leg", action="store_true", help="also run bench.py's C4 leg")
    ap.add_argument("--small", action="store_true", help="C4 scaled to 500 K retained topics / 20 K filters (a rehearsal, not the measurement)")
    args = ap.parse_args()
    if args.lib:
        os.environ["GM_LIB"] = str(Path(args.lib).resolve())
    from rmqtt_b200 import _native as N
    if args.lib:                             # an older build: bind only what it exports
        probe_lib = C.CDLL(os.environ["GM_LIB"])
        for name in [n for n in N.SIGNATURES if not hasattr(probe_lib, n)]:
            del N.SIGNATURES[name]
    import torch
    from rmqtt_b200 import workload as wl
    from rmqtt_b200.engine import Engine

    card = _card()
    cfg = wl.C4.scaled(n_subs=500_000, n_topics=20_000, name="C4-scaled") if args.small else wl.C4
    rb, ro, rv = wl.gen_retained(cfg)
    fb, fo = wl.gen_retain_filters(cfg)
    n = len(fo) - 1
    eng = Engine()
    eng.retain_bulk_load(rb, ro, rv)
    eng.flush()
    lib = N.lib()
    res = eng.retain_match_batch(fb, fo)     # the reference lists: one batch of every filter
    spans, ids = res.spans, res.ids
    out = {"tool": "bench_retain_batcher", "lib": args.lib or "in-tree", "card": card,
           "workload": f"{cfg.name}: {cfg.n_subs} retained topics, {n} SUBSCRIBE filters, seed {cfg.seed:#x}",
           "batch_hits_per_filter": float(spans[:, 1].mean())}

    k = min(args.lone, n)
    cap = int(spans[:k, 1].max()) + 1
    one_spans, one_status = np.zeros((1, 2), np.uint32), np.zeros(1, np.int32)
    one_ids = np.zeros(cap, np.uint32)
    needed = C.c_uint64(0)
    offs1 = np.zeros(2, np.uint32)
    lone = {}
    mismatches = 0
    for graphs in (1, 0):
        eng.debug_knob("small_graphs", graphs)
        lat = np.zeros(k)
        for rep in range(2):                 # the first pass warms up (graph capture, scratch sizes); the second is timed
            t_all = time.perf_counter()
            for i in range(k):
                a, b = int(fo[i]), int(fo[i + 1])
                offs1[1] = b - a
                t = time.perf_counter()
                rc = lib.gm_retain_match_batch(eng._h, fb[a:].ctypes.data, offs1.ctypes.data, 1, one_spans.ctypes.data, one_ids.ctypes.data, cap,
                                               C.byref(needed), one_status.ctypes.data)
                lat[i] = time.perf_counter() - t
                assert rc == 0, (rc, i)
                if rep == 1:
                    got = np.sort(one_ids[:int(one_spans[0, 1])])
                    want = np.sort(ids[spans[i, 0]:spans[i, 0] + spans[i, 1]])
                    mismatches += int(len(got) != len(want) or not (got == want).all())
            wall = time.perf_counter() - t_all
        lone[f"small_graphs_{graphs}"] = {"lookups": k, "p50_us": float(np.percentile(lat, 50) * 1e6), "p99_us": float(np.percentile(lat, 99) * 1e6),
                                          "mean_us": float(lat.mean() * 1e6), "lookups_per_s": k / wall}
    eng.debug_knob("small_graphs", 1)
    out["lone_gm_retain_match_batch"] = lone
    out["lone_lists_equal_batch_lists"] = mismatches == 0
    out["lone_mismatches"] = mismatches

    probe = {}
    if "gm_retain_batcher_probe" in N.SIGNATURES:
        for burst in (1, 64, 2048):
            rounds = args.rounds or max(20, 3000 // burst)
            lt = N.GmLatency()
            rc = lib.gm_retain_batcher_probe(eng._h, fb.ctypes.data, fo.ctypes.data, n, burst, rounds, 0, C.byref(lt))
            probe[f"burst_{burst}"] = lt.as_dict() if rc == 0 else {"error": rc}
    else:
        probe = "not measured: this build has no retained batcher"
    out["retain_batcher_probe"] = probe
    eng.close()

    if args.c4_leg:
        import bench
        dev = torch.device("cuda")
        stream = torch.cuda.current_stream().cuda_stream
        leg = bench._c4_leg(torch, dev, stream, 3.35e12, args.small)
        out["bench_c4_leg"] = {kk: leg[kk] for kk in ("filters_per_s", "ms", "kernel_ms", "count_parity")}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
