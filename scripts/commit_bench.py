#!/usr/bin/env python
"""krag_index_commit on a c3-shaped hybrid index: the incremental merge against a full build of the same rows.

    python scripts/commit_bench.py [--rows 10000000] [--dim 768] [--vocab 1048576] [--terms 2000]

synth_fill 10M device rows (vocab 2^20) and commit (a full build: the index has no base yet).  Then, in turn: add 1, 1,000 and
100,000 rows with host-generated Zipf term lists, committing after each; remove 1 % of the rows at random and commit; compact.
Each commit is timed with a host clock around the synchronous call, beside the phases krag_last_commit reports; the
compaction beside krag_last_compact's.  The bytes a merge moves are counted from the postings (below) and divided by the
commit's wall time: a lower bound of the merge passes' own rate, set against the 3.35 TB/s of the H100 SXM data sheet.

For comparison the index is dropped (two 10M-row indexes do not fit on one card), a fresh one is filled with the same rows
(synth_fill, the same adds and removes) and committed once: a full build of the same live rows.  The postings of sampled terms
(the 50 most frequent and random ones) and a 256-query krag_retrieve, both mapped to node ids, must be bit-identical between
the two.  Prints one JSON line, with the card name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK_GBS = 3350.0
SEED = 20261016


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:
        return {"name": None, "power_limit": None, "error": str(e)}


def host_rows(rng, n, dim, vocab):
    """n rows: unit vectors and Zipf(1.07) term lists of log-normal length (unique ids per row), tf, doc_len"""
    x = rng.standard_normal((n, dim), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    lens = np.clip(np.rint(rng.lognormal(3.2, 0.5, n)), 1, 400).astype(np.int64)
    ids, off = [], [0]
    for k in lens:
        t = np.unique((rng.zipf(1.07, int(k)) - 1) % vocab).astype(np.uint32)
        ids.append(t)
        off.append(off[-1] + t.size)
    tid = np.concatenate(ids)
    tf = rng.integers(1, 4, tid.size).astype(np.uint16)
    off = np.array(off, np.int64)
    dl = (np.add.reduceat(tf.astype(np.int64), off[:-1]) + lens).astype(np.uint32)
    return x, off, tid, tf, dl


def timed_commit(N, ix, vocab, nnz_before):
    t0 = time.perf_counter()
    ix.commit(vocab)
    wall = time.perf_counter() - t0
    lc = N.last_commit()
    nnz = ix.stats().nnz
    # merge passes: survivor count reads doc (4 B / base posting); the merge reads doc + tf (6 B) and writes doc, tf, score
    # (10 B / new posting); the tile index reads doc (4 B / new posting)
    moved = 10 * nnz_before + 14 * nnz if lc["merged"] else None
    return {"commit_s": round(wall, 4), "total_ms": round(lc["total_ms"], 2), "idf_host_ms": round(lc["host_ms"], 2),
            "merged": lc["merged"], "postings_written": lc["postings_written"], "delta_entries": lc["delta_entries"],
            "merge_bytes": moved,
            "merge_gbs_over_commit": round(moved / wall / 1e9, 1) if moved else None,
            "share_of_hbm_peak": round(moved / wall / 1e9 / HBM_PEAK_GBS, 4) if moved else None}, nnz


def snapshot(ix, vocab, terms, q, qt):
    """postings of the sampled terms and a 256-query retrieve, with rows mapped to node ids"""
    post = {}
    n = ix.stats().n_rows
    for t in terms:
        d, s, c = ix.read_postings(int(t), cap=n + 1)
        post[int(t)] = (ix.node_ids(d.astype(np.int64)) if c else np.zeros(0, np.uint64), s.view(np.uint32).copy())
    out = ix.retrieve(q, qt, 10)
    ids = np.zeros(out["ordinal"].shape, np.int64) - 1
    for b, c in enumerate(out["count"]):
        if c:
            ids[b, :c] = ix.node_ids(out["ordinal"][b, :c]).astype(np.int64)
    return post, (ids, out["final"], out["dense"], out["sparse"], out["rank"], out["count"])


def same(a, b):
    pa, ra = a
    pb, rb = b
    ok_post = pa.keys() == pb.keys() and all(np.array_equal(pa[t][0], pb[t][0]) and np.array_equal(pa[t][1], pb[t][1]) for t in pa)
    ok_ret = all(np.array_equal(x, y, equal_nan=x.dtype.kind == "f") for x, y in zip(ra, rb))
    return ok_post, ok_ret


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--vocab", type=int, default=1 << 20)
    ap.add_argument("--terms", type=int, default=2000)
    a = ap.parse_args()
    from kaito_b200 import _native as N
    info = card()
    n, V = a.rows, a.vocab
    rng = np.random.default_rng(SEED)
    adds = []
    next_id = n
    for k in (1, 1000, 100_000):
        adds.append((np.arange(next_id, next_id + k, dtype=np.uint64), host_rows(rng, k, a.dim, V)))
        next_id += k
    all_ids = np.arange(next_id, dtype=np.uint64)
    dead = rng.choice(all_ids, next_id // 100, replace=False).astype(np.uint64)
    q = rng.standard_normal((256, a.dim), dtype=np.float32)
    qt = [np.unique((rng.zipf(1.07, int(rng.integers(2, 8))) - 1) % V).astype(np.uint32) for _ in range(256)]

    ctx = N.Context(device_id=0)
    steps = []
    try:
        extra = sum(len(ids) for ids, _ in adds)
        ix = ctx.create_index("c3", a.dim)
        ix.reserve(n + extra)                    # room for the adds: growing 10M fp32 rows by half would not fit
        ix.synth_fill(n, 0, SEED, V)
        r, nnz = timed_commit(N, ix, V, 0)
        steps.append({"step": "initial commit (full build)", **r})
        for ids, data in adds:
            ix.add(ids, *data)
            r, nnz = timed_commit(N, ix, V, nnz)
            steps.append({"step": f"add {len(ids)} rows", **r})
        ix.remove(dead)
        r, nnz = timed_commit(N, ix, V, nnz)
        steps.append({"step": f"remove {dead.size} rows", **r})
        t0 = time.perf_counter()
        reclaimed = ix.compact()
        wall = time.perf_counter() - t0
        lc = N.last_compact()
        steps.append({"step": "compact", "compact_s": round(wall, 4), "rows_reclaimed": reclaimed,
                      "move_ms": round(lc["move_ms"], 2), "postings_remap_ms": round(lc["postings_ms"], 2),
                      "remap_bytes": 24 * nnz, "remap_gbs": round(24 * nnz / (lc["postings_ms"] / 1e3) / 1e9, 1) if lc["postings_ms"] > 0 else None})
        df = ix.commit_local(V)[0]
        top = np.argsort(df, kind="stable")[-50:]
        terms = np.unique(np.concatenate([top, rng.integers(0, V, a.terms - 50)]))
        merged_out = snapshot(ix, V, terms, q, qt)
        ix.drop()

        F = ctx.create_index("c3_fresh", a.dim)
        F.reserve(n + extra)
        F.synth_fill(n, 0, SEED, V)
        for ids, data in adds:
            F.add(ids, *data)
        F.remove(dead)
        r, _ = timed_commit(N, F, V, 0)
        full = {"step": "full build of the same rows", **r}
        fresh_out = snapshot(F, V, terms, q, qt)
        F.drop()
    finally:
        ctx.close()
    ok_post, ok_ret = same(merged_out, fresh_out)
    print(json.dumps({"metric": "commit", "gpu": info, "rows": n, "dim": a.dim, "vocab": V, "hbm_peak_gbs": HBM_PEAK_GBS,
                      "steps": steps, "full_build": full, "terms_compared": int(terms.size),
                      "postings_identical": bool(ok_post), "retrieve_identical": bool(ok_ret)}))
    if not (ok_post and ok_ret):
        sys.exit(1)


if __name__ == "__main__":
    main()
