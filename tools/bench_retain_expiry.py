#!/usr/bin/env python
"""Retained lookups with deadlines on config C4 (5 M retained topics, 100 K filters from gen_retain_filters), one JSON line.

For 0 %, 10 % and 50 % of the topics carrying a deadline, half of those expired at the time of the lookup (deadlines an hour
before or a day after the wall clock):
  * the device lookup of the whole filter batch through gm_retain_match_batch_device (wall clock): CUDA events around the
    call, median of --reps after one warm-up, with the live hits and the hits without expiry (gm_retain_match_batch_at at 0);
  * the lone-lookup latency through gm_retain_batcher_probe (burst 1), p50 / p99;
  * at 50 %: gm_retain_remove_expired of 1 M expired topics in one call (host time; the removals ship with the next flush),
    and the flush that ships them.
The card's name and power limit are read in the same run.  Usage: python tools/bench_retain_expiry.py [--reps N] [--small]"""
import argparse
import ctypes as C
import json
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
    ap.add_argument("--reps", type=int, default=10, help="timed batch lookups per share")
    ap.add_argument("--small", action="store_true", help="C4 scaled to 500 K retained topics / 20 K filters (a rehearsal, not the measurement)")
    args = ap.parse_args()
    import torch
    from rmqtt_b200 import _native as N
    from rmqtt_b200 import workload as wl
    from rmqtt_b200.engine import Engine

    card = _card()
    cfg = wl.C4.scaled(n_subs=500_000, n_topics=20_000, name="C4-scaled") if args.small else wl.C4
    rb, ro, rv = wl.gen_retained(cfg)
    fb, fo = wl.gen_retain_filters(cfg)
    n = len(fo) - 1
    lib = N.lib()
    out = {"tool": "bench_retain_expiry", "card": card,
           "workload": f"{cfg.name}: {cfg.n_subs} retained topics, {n} SUBSCRIBE filters, seed {cfg.seed:#x}", "shares": {}}
    d_blob = torch.from_numpy(fb).cuda()
    d_offs = torch.from_numpy(fo.view(np.int32)).cuda()
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(0xE5)
    for share in (0.0, 0.1, 0.5):
        now = int(time.time() * 1000)
        dl = np.zeros(len(rv), np.uint64)
        has = rng.random(len(rv)) < share
        expired = has & (rng.random(len(rv)) < 0.5)
        dl[has] = now + 86_400_000
        dl[expired] = now - 3_600_000
        eng = Engine()
        t = time.perf_counter()
        if share:
            eng.retain_bulk_load(rb, ro, rv, dl)
        else:
            eng.retain_bulk_load(rb, ro, rv)
        load_s = time.perf_counter() - t
        eng.flush()
        total = eng.retain_match_batch(fb, fo, now_ms=0).needed          # nothing has expired at time 0
        d_ids = torch.empty(total + 1, dtype=torch.int32, device="cuda")
        times = []
        for rep in range(args.reps + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            live = eng.retain_match_batch_device(d_blob, d_offs, d_spans, d_ids, d_status, stream)
            e1.record()
            torch.cuda.synchronize()
            if rep:
                times.append(e0.elapsed_time(e1))
        lat = N.GmLatency()
        rc = lib.gm_retain_batcher_probe(eng._h, fb.ctypes.data, fo.ctypes.data, n, 1, 3000, 0, C.byref(lat))
        r = {"topics_with_deadline": int(has.sum()), "expired": int(expired.sum()), "bulk_load_s": load_s,
             "batch_ms_median": float(np.median(times)), "batch_ms_min": float(np.min(times)), "hits_live": int(live), "hits_total": int(total),
             "lone_probe": lat.as_dict() if rc == 0 else {"error": rc}}
        if share == 0.5:
            k = min(1_000_000, int(expired.sum()))
            buf = np.empty(k, np.uint32)
            got = C.c_uint64(0)
            t = time.perf_counter()
            rc = lib.gm_retain_remove_expired(eng._h, now, buf.ctypes.data, k, C.byref(got))
            sweep = time.perf_counter() - t
            t = time.perf_counter()
            eng.flush()
            r["remove_expired"] = {"removed": int(got.value), "s": sweep, "flush_s": time.perf_counter() - t, "rc": rc,
                                   "handles_were_expired": bool(expired[buf[:int(got.value)]].all())}
        out["shares"][f"{int(share * 100)}%"] = r
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
