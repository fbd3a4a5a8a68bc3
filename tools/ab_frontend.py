#!/usr/bin/env python
"""Per-kernel device times of the ids-mode match step of C3: the same engine and the same four resident batches as
bench.py's headline leg, one JSON line per configuration on stdout.

Each configuration is timed twice, in runs of their own: the step time with CUDA events and the profiler off, then the
device time of every kernel of the step (k_tokenize, k_bucket_scan, k_bucket_scatter, k_match_fast, k_match_expand,
k_match_slow) from torch.profiler with CUDA activities, averaged per step.  Configurations: the default knobs and
sorted_rows = 0 (k_match_fast reads the token rows through the locality permutation instead of a sorted copy).  The
configurations alternate over `--rounds` rounds.  Every line names the card, its power limit, its SM clock and the active
throttle reasons as read right after that line's timed loop; a final line holds the medians."""
import argparse
import json
import re
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from rmqtt_b200 import workload as wl        # noqa: E402
from rmqtt_b200.engine import Engine         # noqa: E402

KERNELS = ("k_tokenize", "k_bucket_scan", "k_bucket_scatter", "k_match_fast", "k_match_expand", "k_match_slow")
FRONT = KERNELS[:3]


def smi():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks_throttle_reasons.active"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--prof-steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--subs", type=int, default=None)
    ap.add_argument("--topics", type=int, default=None)
    ap.add_argument("--label", default="")
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
    d_ids = torch.empty(64 * n, dtype=torch.int32, device=dev)
    for k in range(len(d_batches)):                  # an output buffer every batch fits, grown the way bench.py grows it
        while True:
            eng.match_batch_device(*d_batches[k], d_spans, d_ids, d_needed, d_status, stream)
            need = int(d_needed.item())
            if need <= d_ids.numel():
                break
            d_ids = torch.empty(int(need * 1.1) + 1024, dtype=torch.int32, device=dev)

    def step(k):
        eng.match_batch_device(*d_batches[k % len(d_batches)], d_spans, d_ids, d_needed, d_status, stream)

    # every configuration sets every knob the configurations vary, so none inherits a value from the one before
    configs = {"default": {"sorted_rows": 1}, "sorted_rows=0": {"sorted_rows": 0}}
    rows = defaultdict(list)
    for rnd in range(args.rounds):
        for name, knobs in configs.items():
            for k, v in knobs.items():
                eng.debug_knob(k, v)
            for k in range(10):
                step(k)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(args.steps):
                step(k)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            card = smi()                                 # clocks and throttle reasons right after this configuration's timed loop
            km = eng.kernel_ms(min(64, args.steps)).mean(axis=0)

            acts = [torch.profiler.ProfilerActivity.CUDA]
            with torch.profiler.profile(activities=acts) as prof:
                for k in range(args.prof_steps):
                    step(k)
                torch.cuda.synchronize()
            per = defaultdict(float)
            for ev in prof.events():
                if ev.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                m = re.search(r"\b(k_\w+?)(<|\(|$)", ev.name)
                if m and m.group(1) in KERNELS:
                    per[m.group(1)] += ev.time_range.elapsed_us() / 1e3 / args.prof_steps     # us -> ms per step
            kern = {k: per.get(k, 0.0) for k in KERNELS}
            row = {"label": args.label, "config": name, "round": rnd, "ms_per_step": ms, "topics_per_s": n / (ms * 1e-3), "gpu": card,
                   "kernel_ms_profiler": kern, "front_end_ms": sum(kern[k] for k in FRONT),
                   "kernel_ms_events": {"k_tokenize+k_bucket_scan+k_bucket_scatter": float(km[0]), "k_match_fast+k_match_expand": float(km[1]),
                                        "k_match_slow": float(km[2])}}
            rows[name].append(row)
            print(json.dumps(row), flush=True)
    summary = {"label": args.label, "summary": cfg.name, "topics": n, "gpu": smi()}
    for name, rs in rows.items():
        summary[name] = {"median_ms_per_step": float(np.median([r["ms_per_step"] for r in rs])),
                         "median_kernel_ms": {k: float(np.median([r["kernel_ms_profiler"][k] for r in rs])) for k in KERNELS}}
    print(json.dumps(summary), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
