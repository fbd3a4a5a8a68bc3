#!/usr/bin/env python
"""The message store (gm_msgstore_*) on C4's topics: 1 M stored messages (gen_retained) with expiry times and store-time marks
for 10 % of them, looked up by 100 K-filter batches (gen_retain_filters), one JSON line.

For each share of already-forwarded queries (0 %, 50 %, 90 %): that share of the batch's queries comes from clients that a
priming call has already served every match of, the rest from clients never seen (fresh keys per repeat, so every repeat
sees the same state).  Per call, median of --reps after one warm-up:
  * walk: the retained lookup of the batch's '+'-appended filters alone (gm_retain_match_batch_device_at on device buffers),
    CUDA events around the call;
  * total: gm_msgstore_get_batch, host buffers in and out, host clock around the call (it ends with a device synchronise);
  * forwarded stage: total - walk (staging, mark checks, batch-order resolution, compaction, marking, copies);
  * the share of matched messages already forwarded, delivered handles and live marks after the run.
Then the lone-get p50: gm_msgstore_get_batch of one filter, host clock, median of 2 000 calls.
The card's name and power limit are read in the same run.  Usage: python tools/bench_msgstore.py [--reps N] [--small]"""
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
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--small", action="store_true", help="100 K messages / 10 K filters (a rehearsal, not the measurement)")
    args = ap.parse_args()
    import torch
    from rmqtt_b200 import _native as N
    from rmqtt_b200 import workload as wl
    from rmqtt_b200.engine import Engine, pack
    from rmqtt_b200.msgstore import NO_SHARE, GpuMessageStore
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    card = _card()
    n_msgs, n_q = (100_000, 10_000) if args.small else (1_000_000, 100_000)
    now = int(time.time() * 1000)
    rng = np.random.default_rng(7)
    blob, offs, handles = wl.gen_retained(wl.C4, n_msgs)
    topics = wl.unpack(blob, offs)
    expiry = now + rng.integers(3_600_000, 7_200_000, n_msgs).astype(np.uint64)
    marked = rng.random(n_msgs) < 0.1
    mo = np.zeros(n_msgs + 1, np.uint32)
    mo[1:] = np.cumsum(marked)
    eng = Engine(max_levels=16)
    ms = GpuMessageStore(eng)
    lib = N.lib()
    t0 = time.perf_counter()
    # store-time marks: subscriber keys 1 000 000 and up (the queries' clients are below)
    cl = (1_000_000 + rng.integers(0, 10_000, int(marked.sum()))).astype(np.uint32)
    sh = np.full(len(cl), NO_SHARE, np.uint32)
    kb, ko = pack(topics)
    ex = np.ascontiguousarray(expiry)
    rc = lib.gm_msgstore_store_batch(ms._h, kb.ctypes.data, ko.ctypes.data, handles.ctypes.data, ex.ctypes.data, n_msgs, mo.ctypes.data, cl.ctypes.data,
                                     sh.ctypes.data)
    assert rc == 0, lib.gm_last_error(None)
    store_s = time.perf_counter() - t0
    fb, fo = wl.gen_retain_filters(wl.C4, n_q)
    filters = wl.unpack(fb, fo)
    # the walk alone: the filters as the store stages them
    wf = [f if (f == b"#" or f.endswith(b"/#")) else f + b"/+" for f in filters]
    wb, wo = pack(wf)
    dev = torch.device("cuda")
    d_blob = torch.from_numpy(np.concatenate([wb, np.zeros(16, np.uint8)])).to(dev)
    d_offs = torch.from_numpy(wo.view(np.int32)).to(dev)
    d_spans = torch.zeros((n_q, 2), dtype=torch.int32, device=dev)
    d_status = torch.zeros(n_q, dtype=torch.int32, device=dev)
    cap_raw = 64 * n_q
    d_ids = torch.zeros(cap_raw, dtype=torch.int32, device=dev)
    raw = C.c_uint64(0)

    def walk():
        s = torch.cuda.current_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        st = lib.gm_retain_match_batch_device_at(eng._h, now, d_blob.data_ptr(), len(wb), d_offs.data_ptr(), n_q, d_spans.data_ptr(), d_ids.data_ptr(), cap_raw,
                                                 C.byref(raw), d_status.data_ptr(), s.cuda_stream)
        e1.record(s)
        e1.synchronize()
        assert st == 0, lib.gm_last_error(None)
        return e0.elapsed_time(e1)

    spans, status = np.zeros((n_q, 2), np.uint32), np.zeros(n_q, np.int32)
    out = np.empty(cap_raw, np.uint32)
    needed = C.c_uint64(0)
    no_share = np.full(n_q, NO_SHARE, np.uint32)

    def get(clients, n=n_q, b=fb, o=fo):
        t = time.perf_counter()
        st = lib.gm_msgstore_get_batch(ms._h, now, b.ctypes.data, o.ctypes.data, n, clients.ctypes.data, no_share.ctypes.data, spans.ctypes.data,
                                       out.ctypes.data, cap_raw, C.byref(needed), status.ctypes.data)
        dt = (time.perf_counter() - t) * 1e3
        assert st == 0, lib.gm_last_error(None)
        return dt

    old = np.arange(n_q, dtype=np.uint32)           # clients 0 .. n_q-1: primed with every match of their query
    get(old)
    walk()
    fresh_base = n_q
    rows = []
    for share in (0.0, 0.5, 0.9):
        sel = rng.random(n_q) < share
        walks, totals, fwd_share = [], [], []
        for rep in range(args.reps + 1):
            clients = np.where(sel, old, fresh_base + np.arange(n_q, dtype=np.uint32)).astype(np.uint32)
            fresh_base += n_q
            w = walk()
            t = get(clients)
            if rep:
                walks.append(w)
                totals.append(t)
                fwd_share.append(1 - needed.value / max(raw.value, 1))
        rows.append({"forwarded_queries": share, "forwarded_matches": round(float(np.median(fwd_share)), 4), "matched": int(raw.value),
                     "delivered": int(needed.value), "walk_ms": round(float(np.median(walks)), 3), "total_ms": round(float(np.median(totals)), 3),
                     "forwarded_stage_ms": round(float(np.median(totals) - np.median(walks)), 3)})
    st = ms.stats()
    lone = []
    one_b, one_o = pack([filters[0]])
    one_c = np.array([0], np.uint32)
    for i in range(2200):
        t = get(one_c, 1, one_b, one_o)
        if i >= 200:
            lone.append(t * 1e3)
    print(json.dumps({"bench": "msgstore", "card": card, "messages": n_msgs, "filters_per_call": n_q, "store_batch_s": round(store_s, 2),
                      "reps": args.reps, "calls": rows, "live_marks": st["marks"], "mark_slots": st["mark_slots"], "rehashes": st["rehashes"],
                      "lone_get_p50_us": round(float(np.median(lone)), 1)}))
    ms.close()
    eng.close()


if __name__ == "__main__":
    main()
