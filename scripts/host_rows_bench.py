#!/usr/bin/env python
"""Device-resident against host-resident fp32 rows (KRAG_ROWS_DEVICE / KRAG_ROWS_HOST) on one GPU.

    python scripts/host_rows_bench.py [--rows 4000000] [--dim 768] [--steps 10] [--warmup 3] [--repeats 2]

Builds the same synthetic hybrid corpus (device-generated rows + Zipf term lists) once per storage mode, then, alternating
the modes, times
  - the dense stage (krag_dev_dense_candidates on device-resident queries, CUDA events on the calling stream), and
  - a hybrid krag_retrieve through the host-buffer API (host clock around the synchronous call),
at batch 256 and P = k * cand_mult = 30.  A separate torch.profiler pass per mode splits the dense stage into the sample
pass, main pass, refine (+ fetch compaction), host rescoring and the fallback scan.  Prints one JSON line with queries/s per
mode, rows fetched from host memory per query, host-link bytes per batch, fallback queries, and the card name and power
limit read in the same call.  Not bench.py: that one measures the default (device) storage only.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:   # the numbers below still stand; say why the card is unknown
        return {"name": None, "power_limit": None, "error": str(e)}


STAGES = [("sample", lambda n: re.search(r"dense_tc_kernel<\d+, \d+, true>", n) is not None),
          ("main", lambda n: "dense_tc_kernel" in n),
          ("refine", lambda n: "refine_kernel" in n or "fetch_compact_kernel" in n),
          ("host_rescore", lambda n: "rescore_mapped_kernel" in n),
          ("device_rescore", lambda n: "rescore_kernel" in n),
          ("fallback_scan", lambda n: "dense_scan_kernel" in n),
          ("fallback_copy", lambda n: "Memcpy HtoD" in n or "memcpy HtoD" in n.lower())]


def stage_ms(prof, steps):
    out = {k: 0.0 for k, _ in STAGES}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        for k, match in STAGES:
            if match(ev.key):
                out[k] += t / 1000.0 / steps
                break
    return {k: round(v, 4) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--vocab", type=int, default=1 << 20)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--cand-mult", type=float, default=3.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=2, help="alternating timed rounds per mode")
    args = ap.parse_args()

    import torch
    from kaito_b200 import _native as N
    assert torch.cuda.is_available(), "needs an H100"
    B, P, dim = args.batch, int(args.k * args.cand_mult), args.dim
    dpad = (dim + 31) // 32 * 32
    g = np.random.default_rng(0)
    modes = {"device": N.ROWS_DEVICE, "host": N.ROWS_HOST}
    setups = {}
    for name, storage in modes.items():
        t0 = time.perf_counter()
        ctx = N.Context(device_id=0, row_storage=storage)
        ix = ctx.create_index(f"hrb_{name}", dim)
        ix.synth_fill(args.rows, 0, 7, args.vocab)
        ix.commit(args.vocab)
        setups[name] = {"ctx": ctx, "ix": ix, "build_s": time.perf_counter() - t0, "index_device_bytes": ix.stats().device_bytes}
    seeds = setups["device"]["ix"].read_rows(0, 1 << 15)
    q = (seeds[g.integers(0, len(seeds), B)] + 0.1 * g.standard_normal((B, dim)) / np.sqrt(dim)).astype(np.float32)
    terms = [list(g.integers(0, 2000, g.integers(3, 9))) for _ in range(B)]
    q_dev = torch.zeros((B, dpad), dtype=torch.float32, device="cuda")
    q_dev[:, :dim] = torch.from_numpy(q).cuda()
    keys = {m: torch.empty((B, P), dtype=torch.int64, device="cuda") for m in modes}
    stream = torch.cuda.current_stream()

    def dense(m, steps):
        ix = setups[m]["ix"]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            ix.dev_dense_candidates(B, q_dev.data_ptr(), P, keys[m].data_ptr(), stream.cuda_stream)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / 1000.0

    def hybrid(m, steps):
        ix = setups[m]["ix"]
        t0 = time.perf_counter()
        for _ in range(steps):
            out = ix.retrieve(q, terms, args.k, cand_mult=args.cand_mult)
        return time.perf_counter() - t0, out

    res = {m: {"dense_s": [], "hybrid_s": [], "fetched": 0, "fallbacks": 0} for m in modes}
    for m in modes:
        dense(m, args.warmup)
        hybrid(m, args.warmup)
    outs = {}
    for _ in range(args.repeats):
        for m in modes:
            f0, fb0 = N.host_rows_fetched(), N.load().krag_tc_fallback_queries()
            res[m]["dense_s"].append(dense(m, args.steps))
            t, outs[m] = hybrid(m, args.steps)
            res[m]["hybrid_s"].append(t)
            res[m]["fetched"] += N.host_rows_fetched() - f0
            res[m]["fallbacks"] += N.load().krag_tc_fallback_queries() - fb0
    same = all(np.array_equal(outs["device"][k], outs["host"][k], equal_nan=True) for k in outs["device"])
    same_dense = bool(torch.equal(keys["device"], keys["host"]))

    stages = {}
    from torch.profiler import ProfilerActivity, profile
    for m in modes:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            dense(m, 3)
        stages[m] = stage_ms(prof, 3)

    n_batches = args.repeats * args.steps * 2          # dense stage + hybrid retrieve per step
    line = {"metric": "host_rows_vs_device_rows", "rows": args.rows, "dim": dim, "batch": B, "P": P, "card": card(),
            "results_identical": bool(same and same_dense)}
    for m in modes:
        r = res[m]
        fetched_per_q = r["fetched"] / (n_batches * B)
        line[m] = {
            "dense_qps": round(B * args.steps / float(np.median(r["dense_s"])), 1),
            "hybrid_qps": round(B * args.steps / float(np.median(r["hybrid_s"])), 1),
            "dense_qps_runs": [round(B * args.steps / s, 1) for s in r["dense_s"]],
            "hybrid_qps_runs": [round(B * args.steps / s, 1) for s in r["hybrid_s"]],
            "fetched_rows_per_query": round(fetched_per_q, 2),
            "host_link_rescore_bytes_per_batch": int(fetched_per_q * B * dpad * 4),
            "fallback_queries": int(r["fallbacks"]),
            "stage_ms_per_dense_batch": stages[m],
            "index_device_bytes": setups[m]["index_device_bytes"],
            "build_s": round(setups[m]["build_s"], 1),
        }
    line["host_pinned_bytes"] = N.host_pinned_bytes()
    print(json.dumps(line), flush=True)
    for m in modes:
        setups[m]["ix"].drop()
        setups[m]["ctx"].close()


if __name__ == "__main__":
    main()
