#!/usr/bin/env python
"""krag_index_compact on a c3-shaped hybrid index, device-resident and host-resident rows.

    python scripts/compact_bench.py [--rows 10000000] [--host-rows 4000000] [--dim 768] [--vocab 1048576] [--steps 5]

Per storage and removal layout (a random pattern, one contiguous run): synth_fill the index, remove 30 % of the rows, commit,
compact; then remove more rows, up to 50 % of the original ones, commit, compact again.  Each compaction is timed with a host
clock around the synchronous call, and its row-move phase with the CUDA events krag_last_compact reports, beside the postings
rebuild.  Hybrid krag_retrieve is timed at batch 256 before and after (queries/s, host clock), and its outputs, mapped to
node ids, must be equal.  Prints one JSON line: per compaction, rows and bytes moved and the move's GB/s (read + write of the
moved bytes) against the 3.35 TB/s of the H100 SXM data sheet, device and pinned bytes before and after; and the card name
and power limit read in the same run.  Host rows default to fewer rows than device rows: 10M x 768 fp32 rows are 30.7 GB of
pinned host memory.  The retrieve outputs go to --out (default: a temporary directory).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK_GBS = 3350.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:
        return {"name": None, "power_limit": None, "error": str(e)}


def retrieve_mapped(ix, q, qt, steps):
    ix.retrieve(q, qt, 10)                       # warm-up of this shape
    t0 = time.perf_counter()
    for _ in range(steps):
        out = ix.retrieve(q, qt, 10)
    dt = (time.perf_counter() - t0) / steps
    ids, fin = np.zeros(out["ordinal"].shape, np.int64) - 1, np.zeros(out["final"].shape)
    for b, c in enumerate(out["count"]):
        if c:
            ids[b, :c] = ix.node_ids(out["ordinal"][b, :c]).astype(np.int64)
            fin[b, :c] = out["final"][b, :c]
    return len(q) / dt, ids, fin


def run_case(N, storage, layout, n, dim, vocab, steps, out_dir):
    ctx = N.Context(device_id=0, row_storage=N.ROWS_HOST if storage == "host" else N.ROWS_DEVICE)
    res = []
    try:
        ix = ctx.create_index("c3", dim)
        ix.synth_fill(n, 0, 20260921, vocab)
        g = np.random.default_rng(1)
        q = g.standard_normal((256, dim), dtype=np.float32)
        qt = [g.integers(0, 4096, 6).astype(np.uint32) for _ in range(256)]
        order = g.permutation(n) if layout == "random" else np.arange(n // 4, n // 4 + n)  % n
        removed = 0
        for frac in (0.3, 0.5):
            k = int(frac * n) - removed
            ix.remove(order[removed:removed + k].astype(np.uint64))
            removed += k
            ix.commit(vocab)
            qps0, ids0, fin0 = retrieve_mapped(ix, q, qt, steps)
            s0, dev0, pin0 = ix.stats(), N.device_bytes(), N.host_pinned_bytes()
            t0 = time.perf_counter()
            reclaimed = ix.compact()
            wall = time.perf_counter() - t0
            rep = N.last_compact()
            s1, dev1, pin1 = ix.stats(), N.device_bytes(), N.host_pinned_bytes()
            qps1, ids1, fin1 = retrieve_mapped(ix, q, qt, steps)
            tag = f"{storage}_{layout}_{int(frac * 100)}"
            np.savez(os.path.join(out_dir, f"retrieve_{tag}.npz"), ids_before=ids0, final_before=fin0, ids_after=ids1, final_after=fin1)
            assert np.array_equal(ids0, ids1) and np.array_equal(fin0, fin1), f"{tag}: retrieve outputs changed"
            move_s = rep["move_ms"] / 1e3
            res.append({
                "storage": storage, "layout": layout, "removed_fraction": frac, "rows_before": s0.n_rows, "rows_after": s1.n_rows,
                "rows_reclaimed": reclaimed, "compact_s": round(wall, 4), "move_ms": round(rep["move_ms"], 3),
                "rows_moved": rep["rows_moved"], "bytes_moved": rep["bytes_moved"],
                "move_gbs": round(2 * rep["bytes_moved"] / move_s / 1e9, 1) if move_s > 0 else None,
                "move_share_of_hbm_peak": round(2 * rep["bytes_moved"] / move_s / 1e9 / HBM_PEAK_GBS, 3) if move_s > 0 else None,
                "postings_rebuild_ms": round(rep["postings_ms"], 1),
                "index_device_bytes": [s0.device_bytes, s1.device_bytes], "process_device_bytes": [dev0, dev1],
                "pinned_bytes": [pin0, pin1], "retrieve_qps_b256": [round(qps0, 1), round(qps1, 1)],
                "outputs_equal": True,
            })
        ix.drop()
    finally:
        ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--host-rows", type=int, default=4_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--vocab", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from kaito_b200 import _native as N
    out_dir = a.out or tempfile.mkdtemp(prefix="compact_bench_")
    os.makedirs(out_dir, exist_ok=True)
    info = card()
    cases = []
    for storage, n in (("device", a.rows), ("host", a.host_rows)):
        for layout in ("random", "contiguous"):
            cases += run_case(N, storage, layout, n, a.dim, a.vocab, a.steps, out_dir)
    print(json.dumps({"metric": "compact", "gpu": info, "dim": a.dim, "vocab": a.vocab, "hbm_peak_gbs": HBM_PEAK_GBS,
                      "outputs": out_dir, "cases": cases}))


if __name__ == "__main__":
    main()
