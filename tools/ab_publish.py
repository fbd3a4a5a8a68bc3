#!/usr/bin/env python
"""Where the ids-mode match step of C3 spends its time: the same engine and batches as bench.py's headline leg, timed in
three forms with CUDA events, one JSON line each on stdout:

  ids          gm_match_batch_device, every matched id written (bench.py `value`)
  no_publish   the same with diag_flags = MP_DIAG_NO_PUBLISH: the walk without writing ids
  desc         descriptor mode (`value_descriptor_mode`): one (ref, cnt) per matched value set instead of its ids

Each line carries the step time and the three kernel_ms columns (tokenise + locality pass, k_match_fast + k_match_expand,
k_match_slow).  The forms alternate over `--rounds` rounds, so a drifting clock shows up as spread rather than as a
difference.  A final line names the card, its power limit and its clocks."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from rmqtt_b200 import workload as wl        # noqa: E402
from rmqtt_b200.engine import Engine         # noqa: E402

MP_DIAG_NO_PUBLISH = 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--subs", type=int, default=None)
    ap.add_argument("--topics", type=int, default=None)
    args = ap.parse_args()
    cfg = wl.C3 if not (args.subs or args.topics) else wl.C3.scaled(n_subs=args.subs, n_topics=args.topics, name="C3-scaled")
    dev = torch.device("cuda")
    stream = torch.cuda.current_stream().cuda_stream

    sb, so, sv = wl.gen_subs(cfg)
    eng = Engine(filters_hint=len(sv))
    eng.bulk_load(sb, so, sv)
    eng.flush()
    del sb, so
    n = cfg.n_topics
    batches = [wl.gen_topics(cfg, n, stream=b) for b in range(args.batches)]
    d_batches = [(torch.from_numpy(tb).to(dev), torch.from_numpy(to.view(np.int32)).to(dev)) for tb, to in batches]
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device=dev)
    d_status = torch.zeros(n, dtype=torch.int32, device=dev)
    d_needed = torch.zeros(1, dtype=torch.int64, device=dev)

    def sized(make, run):   # an output buffer every batch fits, grown the way bench.py grows it
        buf, need_max = make(64 * n), 0
        for k in range(len(d_batches)):
            while True:
                run(k, buf)
                need = int(d_needed.item())
                if need <= buf.shape[0]:
                    break
                buf = make(int(need * 1.1) + 1024)
            need_max = max(need_max, need)
        return buf, need_max

    def ids_step(k, buf):
        eng.match_batch_device(*d_batches[k % len(d_batches)], d_spans, buf, d_needed, d_status, stream)

    def desc_step(k, buf):
        eng.match_batch_device_ex(*d_batches[k % len(d_batches)], d_spans, buf, d_needed, d_status, stream, desc=True)

    d_ids, ids_max = sized(lambda m: torch.empty(m, dtype=torch.int32, device=dev), ids_step)
    d_desc, desc_max = sized(lambda m: torch.empty((m, 2), dtype=torch.int32, device=dev), desc_step)

    forms = {"ids": (0, ids_step, d_ids), "no_publish": (MP_DIAG_NO_PUBLISH, ids_step, d_ids), "desc": (0, desc_step, d_desc)}
    rows = {f: [] for f in forms}
    for rnd in range(args.rounds):
        for name, (flags, fn, buf) in forms.items():
            eng.debug_knob("diag_flags", flags)
            for k in range(5):
                fn(k, buf)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(args.steps):
                fn(k, buf)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            km = eng.kernel_ms(min(64, args.steps)).mean(axis=0)
            row = {"form": name, "round": rnd, "ms_per_step": ms, "topics_per_s": n / (ms * 1e-3),
                   "kernel_ms": {"k_tokenize+k_bucket_scan+k_bucket_scatter": float(km[0]), "k_match_fast+k_match_expand": float(km[1]),
                                 "k_match_slow": float(km[2])}}
            rows[name].append(row)
            print(json.dumps(row), flush=True)
    eng.debug_knob("diag_flags", 0)

    def med(name, key):
        v = [r["ms_per_step"] if key is None else r["kernel_ms"][key] for r in rows[name]]
        return float(np.median(v))

    fast = "k_match_fast+k_match_expand"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"summary": cfg.name, "topics": n, "ids_needed_max": ids_max, "descs_needed_max": desc_max,
                      "median_ms_per_step": {f: med(f, None) for f in forms}, "median_match_ms": {f: med(f, fast) for f in forms},
                      "publish_ms": med("ids", fast) - med("no_publish", fast), "gpu": smi}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
