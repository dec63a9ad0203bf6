"""ColBERT reranking from stored passage vectors against encoding every candidate in the call, at the colbertv2.0 shape
(12 x 768, dim 128) and the answerai-colbert-small shape (12 x 384, dim 96), random weights, 256 queries x N distinct
candidates of a fixed token count (the inputs of scripts/colbert_bench.py: 15 % of passage rows on the skiplist).  Per point
and precision mode:
  - krag_late_rerank_stored (every candidate stored) and krag_late_rerank, alternating, median of --reps synchronised calls;
    their positions and scores must be equal at every timed call;
  - maxsim_kernel alone: torch.profiler CUDA time in one stored call, in a run of its own after the timing, with the bytes
    (every pair's kept rows, read once) and FMA count from the shapes, the achieved rates, and the share of the bound
    max(bytes / 3.35 TB/s, FMAs / (67 TFLOP/s / 2)) -- the data sheet's HBM3 bandwidth and dense FP32 rate;
  - append throughput: passages / s and stored bytes per passage of krag_late_store_append over the call's passages.
Every row carries the card's name, power limit and max SM clock read in this call.  Prints one JSON line per point.

  python scripts/colbert_store_bench.py [--shapes colbertv2.0,answerai-colbert-small] [--n 10,30] [--lens 128,180] [--reps 3]
                                        [--out file]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

HBM_BPS, FP32_FMA_PER_S = 3.35e12, 67e12 / 2


def maxsim_ms(e, store, args):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.late_rerank_stored(store, *args)
    us = [getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
          for ev in prof.key_averages() if "maxsim_kernel" in ev.key]
    return float(sum(us)) / 1e3 if us else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="colbertv2.0,answerai-colbert-small")
    ap.add_argument("--n", default="10,30")
    ap.add_argument("--lens", default="128,180")
    ap.add_argument("--queries", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="fp32,fp16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    modes = a.precision.split(",")
    if not modes or any(m not in ("fp32", "fp16") for m in modes) or a.reps < 1:
        ap.error("--precision takes fp32, fp16 or both; --reps >= 1")
    from colbert_bench import QL, inputs
    from kaito_b200 import _native
    from tests.test_gpu_colbert import SHAPES, _model, _state
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if not gpu:
        raise SystemExit("colbert_store_bench: no GPU (nvidia-smi reports none); every number here is a GPU measurement")
    ctx = _native.Context(device_id=0)
    rows = []
    for shape in [s for s in a.shapes.split(",") if s]:
        cfg, state, w = _state(*SHAPES[shape], "bench")
        dim = SHAPES[shape][1]
        e = _model(ctx, cfg, state, w)
        e.set_store_budget(16 << 30)
        for n in map(int, a.n.split(",")):
            for plen in map(int, a.lens.split(",")):
                g = np.random.default_rng(n + plen)
                q, keys, p_ids, d_off, keep, poff, pp = inputs(g, a.queries, n, plen)
                call = (q, keys, p_ids, d_off, keep, poff, pp, 10)
                empty = (np.zeros(0, np.int32), np.zeros(1, np.int32), np.zeros(0, np.uint8))
                kept = int(keep.sum())
                row = {"model": shape, "queries": a.queries, "N": n, "passage_tokens": plen, "pairs": int(poff[-1]),
                       "kept_rows": kept, "query_rows": a.queries * QL}
                for mode in modes:
                    sfx = "" if mode == "fp32" else "_fp16"
                    e.set_precision(mode)
                    s = _native.LateStore(e)
                    t0 = time.perf_counter()
                    got = s.append(p_ids, d_off, keep)                      # returns synchronised
                    t_app = time.perf_counter() - t0
                    assert got.all()
                    st = s.stats()
                    stored = (q, keys, *empty, poff, pp, 10)               # passage p is ordinal p
                    for _ in range(2):                                     # warm-up (graphs are captured on the second sight)
                        e.late_rerank(*call); e.late_rerank_stored(s, *stored)
                    t_call, t_store = [], []
                    for _ in range(a.reps):
                        t0 = time.perf_counter()
                        want = e.late_rerank(*call)
                        t_call.append(time.perf_counter() - t0)
                        t0 = time.perf_counter()
                        have = e.late_rerank_stored(s, *stored)
                        t_store.append(time.perf_counter() - t0)
                        assert np.array_equal(want[0], have[0]) and np.array_equal(want[1], have[1], equal_nan=True), (shape, n, plen, mode)
                    ms = maxsim_ms(e, s, stored)
                    nbytes, fmas = 4.0 * kept * dim, float(QL) * kept * dim      # each pair: its query's QL rows x its kept rows
                    bound_ms = max(nbytes / HBM_BPS, fmas / FP32_FMA_PER_S) * 1e3
                    row.update({f"per_call{sfx}_ms": float(np.median(t_call)) * 1e3, f"stored{sfx}_ms": float(np.median(t_store)) * 1e3,
                                f"maxsim_kernel{sfx}_ms": ms, f"maxsim{sfx}_gb_per_s": nbytes / (ms * 1e-3) / 1e9 if ms else None,
                                f"maxsim{sfx}_tflops": 2 * fmas / (ms * 1e-3) / 1e12 if ms else None,
                                f"maxsim{sfx}_bound_ms": bound_ms, f"maxsim{sfx}_share_of_bound": bound_ms / ms if ms else None,
                                f"append{sfx}_passages_per_s": (len(d_off) - 1) / t_app,
                                f"stored_bytes{sfx}_per_passage": st["rows"] * dim * 4 / st["stored"],
                                f"store{sfx}_device_bytes": st["device_bytes"]})
                    s.destroy()
                row["gpu"] = gpu
                print(json.dumps(row), flush=True)
                rows.append(row)
        e.destroy()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
