"""Compaction of the multi-GPU service's round-robin shards at service scale (ShardedRetriever.compact, kaito_rag.h
krag_redeal_begin): a hybrid corpus as G round-robin shards, 30 % of the rows removed, compacted, then up to 50 % and
compacted again.  Reports per compaction the wall time, the row-move time (CUDA events, first pack to finish, of one
shard) and the BM25 rebuild (the commit that ends it), the payload moved and its rate, device and pinned bytes before and
after, retrieve queries/s before (tombstoned) and after, and whether the results are equal once the new ordinals are
mapped back to the old ones.  The card's name and power limit are read in the same run.

  one GPU:        python scripts/sharded_compact_bench.py            (G shards in one process, one thread per rank)
  several GPUs:   torchrun --nproc-per-node G scripts/sharded_compact_bench.py   (one shard per GPU, NCCL)

Rows come from krag_synth_fill (dense, generated on the device) and the oracle's Zipf term lists (--mean-len tokens per
row), added round robin so that node id = global ordinal, as the service deals them."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kaito_b200 import _native, sharded  # noqa: E402
from kaito_b200.sharded import NativeStages, ShardedRetriever  # noqa: E402
from oracle import oracle as o  # noqa: E402

HBM_TBPS = 3.35     # H100 SXM data sheet


class _Group:
    def __init__(self, rank, shared):
        self.rank, self.shared = rank, shared


class Loopback:
    """torch.distributed for G threads of one process on one GPU: every thread issues on the legacy default stream, so a
    barrier orders each rank's kernels before the copies that read their output"""

    def __init__(self, world):
        self.world, self.barrier, self.slots = world, threading.Barrier(world), [None] * world

    @staticmethod
    def is_initialized():
        return True

    @staticmethod
    def get_world_size(group=None):
        return group.shared.world

    @staticmethod
    def get_rank(group=None):
        return group.rank

    @staticmethod
    def all_reduce(t, group=None):
        sh = group.shared
        torch.cuda.current_stream(t.device).synchronize()
        sh.slots[group.rank] = t.detach().cpu().clone()
        sh.barrier.wait()
        total = sum(sh.slots[1:], sh.slots[0].clone())
        sh.barrier.wait()
        t.copy_(total.to(t.device))

    @staticmethod
    def all_gather_into_tensor(out, inp, group=None):
        sh = group.shared
        sh.slots[group.rank] = inp
        sh.barrier.wait()
        n = inp.numel()
        for r in range(sh.world):
            out.view(-1)[r * n:(r + 1) * n].copy_(sh.slots[r].reshape(-1))
        sh.barrier.wait()

    @staticmethod
    def all_to_all_single(out, inp, output_split_sizes=None, input_split_sizes=None, group=None):
        sh = group.shared
        sh.slots[group.rank] = (inp, [int(x) for x in input_split_sizes])
        sh.barrier.wait()
        off = 0
        for t in range(sh.world):
            tin, splits = sh.slots[t]
            a, n = sum(splits[:group.rank]), splits[group.rank]
            if n:
                out[off:off + n].copy_(tin[a:a + n])
            off += n
        sh.barrier.wait()


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def build(ctx, shards, G, a, lens_out):
    """rows [0, n) in chunks: dense from krag_synth_fill on a scratch index, terms from the oracle; shard s of `shards` gets
    the rows o with o % G == s, node id o"""
    gen_rows = []
    for c in range(0, a.n, a.chunk):
        m = min(a.chunk, a.n - c)
        gen = ctx.create_index("gen", a.dim)
        gen.synth_fill(m, row_base=c, seed=a.seed)
        x = gen.read_rows(0, m)
        gen.drop()
        off, tid, tf, dl = o.synth_sparse(m, a.vocab, a.seed + c, mean_len=a.mean_len)
        lens_out[c:c + m] = np.diff(off)
        ords = c + np.arange(m)
        for s, ix in shards.items():
            i = np.nonzero(ords % G == s)[0]
            lens = np.diff(off)[i]
            noff = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
            take = np.repeat(off[i] - noff[:-1], lens) + np.arange(noff[-1], dtype=np.int64)
            ix.add(ords[i].astype(np.uint64), x[i], noff, tid[take], tf[take], dl[i])
        if c == 0:
            gen_rows = x[:a.queries // 2].copy()
    return gen_rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--shards", type=int, default=4, help="shards on one GPU (ignored under torchrun: one per rank)")
    ap.add_argument("--vocab", type=int, default=1 << 20)
    ap.add_argument("--mean-len", type=float, default=32.0)
    ap.add_argument("--chunk", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=256)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--window-rows", type=int, default=0, help="0: ShardedRetriever.COMPACT_WINDOW_ROWS")
    ap.add_argument("--seed", type=int, default=20260921)
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    multi = int(os.environ.get("WORLD_SIZE", "1")) > 1
    if multi:
        from kaito_b200.sharded_engine import init_distributed
        rank, G, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
        init_distributed(rank, G, lr, int(os.environ["MASTER_PORT"]))
        ranks, dev_id = [rank], lr
    else:
        G, ranks, dev_id = a.shards, list(range(a.shards)), 0
        shared = Loopback(G)
        sharded.dist = shared
        os.environ["KRAG_P2P"] = "0"
    ctx = _native.Context(device_id=dev_id)
    dev = torch.device("cuda", dev_id)
    shards = {s: ctx.create_index(f"shard{s}", a.dim) for s in ranks}
    for s, ix in shards.items():
        ix.reserve(a.n // G + 1)
    lens = np.zeros(a.n, np.int64)
    t0 = time.time()
    qrows = build(ctx, shards, G, a, lens)
    build_s = time.time() - t0
    for s, ix in shards.items():
        ix.set_ordinal_map(s, G)
    dpad = next(iter(shards.values())).stats().dim_padded
    srs = {s: ShardedRetriever(NativeStages(ctx, ix), dev, dpad, group=_Group(s, shared) if not multi else None)
           for s, ix in shards.items()}

    def on_ranks(fn):
        """fn(rank) on every rank this process serves (threads on one GPU)"""
        if multi:
            return [fn(ranks[0])]
        res, err = [None] * G, []

        def body(r):
            try:
                res[r] = fn(r)
            except BaseException as e:
                err.append(e)
                shared.barrier.abort()
        th = [threading.Thread(target=body, args=(r,)) for r in ranks]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if err:
            raise err[0]
        return res

    def n_rows(s):
        return int(shards[s].stats().n_rows)

    on_ranks(lambda s: srs[s].commit(a.vocab, n_rows(s), ordinal_base=s))
    rng = np.random.default_rng(a.seed)
    q = np.concatenate([qrows + 0.05 * rng.standard_normal(qrows.shape).astype(np.float32),
                        rng.standard_normal((a.queries - len(qrows), a.dim)).astype(np.float32)])
    q = np.ascontiguousarray(q / np.linalg.norm(q, axis=1, keepdims=True), np.float32)
    qs = o.synth_query_terms(a.vocab, a.queries, a.seed + 1, rank_offset=100)

    def retrieve():
        outs = on_ranks(lambda s: srs[s].retrieve(q, qs, a.k))
        torch.cuda.synchronize(dev)
        return outs[0]

    def qps():
        retrieve()
        t = time.time()
        for _ in range(a.iters):
            out = retrieve()
        return a.queries * a.iters / (time.time() - t), out

    live = np.ones(a.n, bool)
    ords = np.arange(a.n)                 # current ordinal -> original row
    report = {"card": card(), "shards": G, "gpus": G if multi else 1, "n": a.n, "dim": a.dim, "vocab": a.vocab,
              "mean_len": a.mean_len, "build_s": round(build_s, 1), "steps": []}
    for target in (0.3, 0.5):
        cur = len(ords)
        n_rm = int(round(a.n * target)) - (a.n - cur)
        rm = np.sort(rng.choice(cur, n_rm, replace=False))
        for s, ix in shards.items():
            mine = rm[rm % G == s]
            ix.remove(mine.astype(np.uint64))
        on_ranks(lambda s: srs[s].commit(a.vocab, n_rows(s), ordinal_base=s))
        qps_before, out_before = qps()
        keep = np.ones(cur, bool)
        keep[rm] = False
        first = int(rm[0]) if len(rm) else cur
        moving = np.flatnonzero(keep)[np.flatnonzero(keep) >= first]      # live rows whose ordinal changes
        dev0, pin0 = _native.device_bytes(), _native.host_pinned_bytes()
        torch.cuda.synchronize(dev)
        t = time.time()
        res = on_ranks(lambda s: srs[s].compact(a.vocab, window_rows=a.window_rows or None))
        torch.cuda.synchronize(dev)
        wall = time.time() - t
        comp, commit = _native.last_compact(), _native.last_commit()
        dev1, pin1 = _native.device_bytes(), _native.host_pinned_bytes()
        qps_after, out_after = qps()
        # new ordinal j was old ordinal np.flatnonzero(keep)[j]
        old_of_new = np.flatnonzero(keep)
        mapped = dict(out_after)
        od = out_after["ordinal"]
        mapped["ordinal"] = np.where(od >= 0, old_of_new[np.maximum(od, 0)], -1)
        equal = all(np.array_equal(mapped[k], out_before[k], equal_nan=True) for k in out_before)
        payload = len(moving) * (32 + dpad * 4) + int(lens[ords[moving]].sum()) * 8     # row payloads + 8 B per term entry
        ords = ords[keep]
        move_s = comp["move_ms"] / 1e3
        step = {"removed_fraction": target, "rows_before": cur, "rows_after": len(ords), "reclaimed": int(res[0][0]),
                "wall_s": round(wall, 3), "move_ms_one_shard": round(comp["move_ms"], 1), "rebuild_commit_ms": round(commit["total_ms"], 1),
                "rows_moved": int(len(moving)), "payload_bytes": payload,
                "payload_GBps": round(payload / move_s / 1e9, 1) if move_s > 0 else None,
                "device_bytes_before": dev0, "device_bytes_after": dev1, "pinned_bytes_before": pin0, "pinned_bytes_after": pin1,
                "qps_before": round(qps_before, 1), "qps_after": round(qps_after, 1), "equal_mapped": bool(equal)}
        if not multi and move_s > 0:   # pack, the exchange copy and unpack each read and write the payload in HBM
            step["hbm_bytes_est"] = 6 * payload
            step["hbm_share_of_3.35TBps"] = round(6 * payload / move_s / (HBM_TBPS * 1e12), 3)
        report["steps"].append(step)
    if not multi or ranks[0] == 0:
        line = json.dumps(report)
        print(line, flush=True)
        if a.out:
            with open(a.out, "w") as f:
                f.write(line + "\n")
    for ix in shards.values():
        ix.drop()
    ctx.close()


if __name__ == "__main__":
    main()
