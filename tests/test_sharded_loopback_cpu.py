"""The in-process stand-in for torch.distributed that tests/test_gpu_shards_one_device.py drives G shards on one GPU
with: run with threads over the oracle-backed stages of tests/test_sharded_cpu.py, the sharded pipeline must equal the
single-shard oracle pipeline exactly, as it does under gloo with one process per rank."""
import numpy as np
import pytest
import torch

from tests.test_gpu_shards_one_device import Loopback, run_ranks
from tests.test_sharded_cpu import OracleStages


@pytest.mark.parametrize("world,n,layout", [(2, 2001, "contiguous"), (3, 1000, "contiguous"), (3, 1000, "round_robin"),
                                            (8, 5, "round_robin")])
def test_loopback_shards_equal_single_shard_oracle(oracle, monkeypatch, world, n, layout):
    from kaito_b200 import sharded
    monkeypatch.setattr(sharded, "dist", Loopback)
    o = oracle
    d, vocab, k, B = 48, 300, 7, 5
    x = o.synth_dense(n, d, 1)
    off, ids, tf, dl = o.synth_sparse(n, vocab, 2)
    q = o.synth_queries(x, B, 3)
    qs = o.synth_query_terms(vocab, B, 4, rank_offset=20)

    def rank_fn(rank, group):
        rows = (np.arange(rank, n, world) if layout == "round_robin"
                else np.arange(*sharded.shard_range(n, world, rank)))
        lens = off[rows + 1] - off[rows]
        loff = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        idx = np.repeat(off[rows] - loff[:-1], lens) + np.arange(loff[-1], dtype=np.int64)
        stages = OracleStages(o, x[rows], (loff, ids[idx], tf[idx], dl[rows]), vocab)
        if layout == "round_robin":
            # global ordinal of local row r is rank + r * world: the oracle stages number rows contiguously, so map back
            stages.dense_candidates = _strided(stages.dense_candidates, 2, rank, world)
            stages.bm25_candidates = _strided(stages.bm25_candidates, 4, rank, world)
        sr = sharded.ShardedRetriever(stages, torch.device("cpu"), d, group=group)
        n_docs, total, base = sr.commit(vocab, len(rows), ordinal_base=0 if layout == "round_robin" else None)
        assert (n_docs, total) == (n, int(dl.astype(np.int64).sum()))
        got = sr.retrieve(q, qs, k)
        sr_v = sharded.ShardedRetriever(OracleStages(o, x[rows], None, vocab), torch.device("cpu"), d, group=group)
        sr_v.stages.base = base
        if layout == "round_robin":
            sr_v.stages.dense_candidates = _strided(sr_v.stages.dense_candidates, 2, rank, world)
        return got, sr_v.retrieve(q, None, k)

    outs = run_ranks(world, rank_fn)
    post = o.bm25_build(off, ids, tf, dl, vocab)
    P = o.pool_size(k)
    for got, got_v in outs:
        for b in range(B):
            dd, do = o.dense_topk(x, q[b:b + 1], P)
            bs, bo = o.bm25_query(post, qs[b], P)
            fin, de, sp, rk, od = o.fuse(dd[0], do[0], bs, bo, k)
            c = int(got["count"][b])
            assert c == len(od)
            assert np.array_equal(got["ordinal"][b, :c], od) and np.array_equal(got["final"][b, :c], fin)
            assert np.array_equal(got["rank"][b, :c], rk)
            kv = min(k, int((do[0] >= 0).sum()))
            assert int(got_v["count"][b]) == kv and np.array_equal(got_v["ordinal"][b, :kv], do[0, :kv])


def _strided(fn, out_arg, rank, world):
    """wrap an OracleStages candidate stage (base 0) so that its keys carry the ordinal rank + row * world; the stage
    writes its output keys to positional argument `out_arg`"""
    def wrapped(*args):
        out = args[out_arg]
        fn(*args)
        keys = out.numpy().view(np.uint64)
        live = keys != np.uint64(0xFFFFFFFFFFFFFFFF)
        lo = keys & np.uint64(0xFFFFFFFF)
        keys[live] = (keys[live] & ~np.uint64(0xFFFFFFFF)) | (lo[live] * np.uint64(world) + np.uint64(rank))
    return wrapped
