#!/usr/bin/env python
"""Round-2 A/B measurements on one GPU (C3): tokeniser with / without the TMA bulk stage, e2e chunk size,
and the retained lookup (C4) with work counters.  One JSON line per measurement on stdout."""
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from rmqtt_b200 import _native as N          # noqa: E402
from rmqtt_b200 import workload as wl        # noqa: E402
from rmqtt_b200.engine import Engine         # noqa: E402

dev = torch.device("cuda")
stream = torch.cuda.current_stream().cuda_stream
lib = N.lib()


def c3(which):
    cfg = wl.C3
    sb, so, sv = wl.gen_subs(cfg)
    eng = Engine(filters_hint=cfg.n_subs)
    eng.bulk_load(sb, so, sv)
    eng.flush()
    n = cfg.n_topics
    hb = [wl.gen_topics(cfg, n, stream=b) for b in range(4)]
    db = [(torch.from_numpy(tb).to(dev), torch.from_numpy(to.view(np.int32)).to(dev)) for tb, to in hb]
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device=dev)
    d_status = torch.zeros(n, dtype=torch.int32, device=dev)
    d_needed = torch.zeros(1, dtype=torch.int64, device=dev)
    d_ids = torch.empty(64 * n, dtype=torch.int32, device=dev)
    if "tok" in which:
        for bulk in (0, 1, 0, 1):
            eng.debug_knob("tok_bulk", bulk)
            for k in range(25):
                eng.match_batch_device(*db[k % 4], d_spans, d_ids, d_needed, d_status, stream)
            torch.cuda.synchronize()
            k = eng.kernel_ms(20).mean(axis=0)
            print(json.dumps({"ab": "k_tokenize bulk stage (cp.async.bulk -> smem)", "tok_bulk": bulk, "tokenize+sort_ms": float(k[0]), "k_match_fast_ms": float(k[1])}), flush=True)
    if "e2e" in which:
        need = C.c_uint64(0)
        pins = []

        def pin(nbytes):
            p = lib.gm_host_alloc_near(eng._h, nbytes); pins.append(p); return p

        p_in = []
        for tb, to in hb:
            pb, po = pin(len(tb)), pin(4 * (n + 1))
            C.memmove(pb, tb.ctypes.data, len(tb)); C.memmove(po, to.ctypes.data, 4 * (n + 1))
            p_in.append((pb, po))
        cap = 8 * n
        p_spans, p_status, p_desc = pin(8 * n), pin(4 * n), pin(8 * cap)
        for chunk in (32768, 65536, 131072, 262144, 1 << 20):
            eng.debug_knob("e2e_chunk", chunk)
            for k in range(3):
                assert lib.gm_match_batch_desc(eng._h, *p_in[k % 4], n, p_spans, p_desc, cap, C.byref(need), p_status) == 0
            t0 = time.perf_counter()
            for k in range(12):
                assert lib.gm_match_batch_desc(eng._h, *p_in[k % 4], n, p_spans, p_desc, cap, C.byref(need), p_status) == 0
            dt = (time.perf_counter() - t0) / 12
            print(json.dumps({"ab": "e2e descriptor mode, pipeline chunk", "chunk_topics": chunk, "ms_per_step": dt * 1e3, "topics_per_s": n / dt}), flush=True)
    eng.close()


def c4():
    cfg = wl.C4
    rb, ro, rv = wl.gen_retained(cfg)
    fb, fo = wl.gen_retain_filters(cfg)
    n = len(fo) - 1
    eng = Engine()
    eng.retain_bulk_load(rb, ro, rv)
    eng.flush()
    d_blob, d_offs = torch.from_numpy(fb).to(dev), torch.from_numpy(fo.view(np.int32)).to(dev)
    d_spans = torch.zeros((n, 2), dtype=torch.int32, device=dev)
    d_status = torch.zeros(n, dtype=torch.int32, device=dev)
    d_ids = torch.empty(8 << 20, dtype=torch.int32, device=dev)
    for _ in range(13):
        hits = eng.retain_match_batch_device(d_blob, d_offs, d_spans, d_ids, d_status, stream)
    torch.cuda.synchronize()
    k = eng.kernel_ms(10).mean(axis=0)
    print(json.dumps({"ab": "retained lookup C4 (task rounds + in-thread literal chains + child masks)", "filters": n, "hits": hits,
                      "tokenize_ms": float(k[0]), "walk_ms": float(k[1]), "publish_ms": float(k[2]), "filters_per_s": n / (float(k.sum()) * 1e-3)}), flush=True)
    eng.close()


if __name__ == "__main__":
    which = sys.argv[1:] or ["tok", "e2e", "c4"]
    if "c4" in which:
        c4()
    if "tok" in which or "e2e" in which:
        c3(which)
