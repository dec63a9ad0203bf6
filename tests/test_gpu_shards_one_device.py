"""The multi-shard /retrieve on one GPU: G shard indexes in one context, driven by the production ShardedRetriever
(kaito_b200.sharded) with one thread per rank and an in-process stand-in for torch.distributed.

Every case compares two ways:
  (a) with the oracle pipeline over the whole corpus (dense_topk, bm25_build, bm25_query, fuse): ids, finals, ranks,
      dense and sparse scores exactly;
  (b) with one index that holds every row, through Index.retrieve: every output array bit for bit (DESIGN section 5:
      the sharded results equal the single-GPU service's, ties included).
KRAG_P2P=0 keeps the data path on all-gather -> krag_dev_merge (the peer-memory exchange needs one process per GPU)."""
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

PAD = np.uint64(0xFFFFFFFFFFFFFFFF)
M32 = np.uint64(0xFFFFFFFF)


# ------------------------------------------------------------------------------------------- loopback distributed
class LoopbackGroup:
    """what one rank passes as `group`: its rank and the exchange state shared by the G ranks"""

    def __init__(self, rank, shared):
        self.rank, self.shared = rank, shared


class _Shared:
    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=600)
        self.slots = [None] * world


class Loopback:
    """torch.distributed for G threads of one process.  Every thread issues on the same (legacy default) CUDA stream, so
    the barrier orders each rank's kernels before the copies that read their output."""

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
        """sum; the stream is synchronised and the reduction done on the host, in rank order"""
        sh = group.shared
        if t.is_cuda:
            torch.cuda.current_stream(t.device).synchronize()
        sh.slots[group.rank] = t.detach().cpu().clone()
        sh.barrier.wait()
        total = sh.slots[0].clone()
        for r in range(1, sh.world):
            total += sh.slots[r]
        sh.barrier.wait()                      # every rank has read the slots before they can be reused
        t.copy_(total.to(t.device))

    @staticmethod
    def all_gather_into_tensor(out, inp, group=None):
        """concatenation along dim 0; copies run on the current stream"""
        sh = group.shared
        sh.slots[group.rank] = inp
        sh.barrier.wait()
        n = inp.numel()
        flat = out.view(-1)
        for r in range(sh.world):
            flat[r * n:(r + 1) * n].copy_(sh.slots[r].reshape(-1))
        sh.barrier.wait()


def run_ranks(world, fn):
    """fn(rank, group) on `world` threads; returns the per-rank results, re-raises the first failure"""
    shared = _Shared(world)
    res, err = [None] * world, [None] * world

    def body(r):
        try:
            res[r] = fn(r, LoopbackGroup(r, shared))
        except BaseException as e:     # a failed rank must not leave its peers waiting at a barrier
            err[r] = e
            shared.barrier.abort()

    ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    first = [e for e in err if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if first or any(e is not None for e in err):
        raise (first or [e for e in err if e is not None])[0]
    return res


@pytest.fixture
def loopback(monkeypatch):
    from kaito_b200 import sharded
    monkeypatch.setattr(sharded, "dist", Loopback)
    monkeypatch.setenv("KRAG_P2P", "0")
    return sharded


# ------------------------------------------------------------------------------------------------------ helpers
def sub_csr(csr, rows):
    """term lists of `rows` (in that order) as a CSR of their own"""
    off, ids, tf, dl = csr
    rows = np.asarray(rows, np.int64)
    lens = off[rows + 1] - off[rows]
    noff = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = np.repeat(off[rows] - noff[:-1], lens) + np.arange(noff[-1], dtype=np.int64)
    return noff, ids[idx], tf[idx], dl[rows]


def live_csr(csr, live):
    """the CSR with the term lists of dead rows emptied (row numbering kept)"""
    off, ids, tf, dl = csr
    keep = np.repeat(live, np.diff(off))
    noff = np.concatenate([[0], np.cumsum(np.where(live, np.diff(off), 0))]).astype(np.int64)
    return noff, ids[keep], tf[keep], dl


def global_stats(csr, live, vocab):
    off, ids, tf, dl = csr
    keep = np.repeat(live, np.diff(off))
    df = np.bincount(ids[keep], minlength=vocab).astype(np.uint32)
    return df, int(live.sum()), int(dl[live].astype(np.int64).sum())


def bitmap(mask):
    return np.packbits(np.concatenate([mask, np.zeros((-len(mask)) % 32, bool)]), bitorder="little").view(np.uint32).copy()


class Shards:
    """G shard indexes in one context, each with its ShardedRetriever (one per rank, as on G GPUs)"""

    def __init__(self, sharded, ctx, name, x, csr, vocab, G, layout):
        from kaito_b200.sharded import NativeStages, shard_range
        self.G, self.vocab, self.layout = G, vocab, layout
        n = x.shape[0]
        if layout == "round_robin":       # the service deals row g to shard g % G
            self.rows = [np.arange(s, n, G) for s in range(G)]
        else:                             # the bench: contiguous ranges
            self.rows = [np.arange(*shard_range(n, G, s)) for s in range(G)]
        self.ix, self.stages = [], []
        for s in range(G):
            ix = ctx.create_index(f"{name}_{s}", x.shape[1])
            r = self.rows[s]
            if len(r):
                ix.add(r.astype(np.uint64), x[r], *sub_csr(csr, r))
            if layout == "round_robin":
                ix.set_ordinal_map(s, G)
            self.ix.append(ix)
            self.stages.append(NativeStages(ctx, ix))
        dpad = self.ix[0].stats().dim_padded
        self.sr = [None] * G

        def mk(rank, group):
            self.sr[rank] = sharded.ShardedRetriever(self.stages[rank], torch.device("cuda", 0), dpad, group=group)
        run_ranks(G, mk)

    def commit(self):
        def fn(rank, group):
            self.sr[rank].group = group
            n_local = len(self.rows[rank])
            if self.layout == "round_robin":
                return self.sr[rank].commit(self.vocab, n_local, ordinal_base=rank)
            return self.sr[rank].commit(self.vocab, n_local)
        return run_ranks(self.G, fn)

    def remove(self, node_ids):
        for s, ix in enumerate(self.ix):
            mine = np.intersect1d(np.asarray(node_ids, np.int64), self.rows[s])
            assert ix.remove(mine.astype(np.uint64)) == len(mine)

    def retrieve(self, q, qs, k, **kw):
        def fn(rank, group):
            self.sr[rank].group = group
            return self.sr[rank].retrieve(q, qs, k, **kw)
        outs = run_ranks(self.G, fn)
        for o in outs[1:]:               # every rank ends with the same result
            for name in o:
                assert np.array_equal(o[name], outs[0][name], equal_nan=True), name
        return outs[0]

    def drop(self):
        for ix in self.ix:
            ix.drop()


def assert_same(got, ref, what):
    for name in ("count", "ordinal", "final", "dense", "sparse", "rank"):
        a, b = got[name], ref[name]
        if a.dtype.kind == "f":
            a, b = a.view(np.uint64 if a.itemsize == 8 else np.uint32), b.view(np.uint64 if b.itemsize == 8 else np.uint32)
        assert np.array_equal(a, b), (what, name, np.nonzero((a != b).reshape(len(a), -1).any(axis=-1))[0][:5].tolist())


class OracleRef:
    """the single-index oracle pipeline over the whole corpus for one alive state; candidate lists computed once at the
    largest pool (a top-P list is a prefix of every longer one: the order is total)"""

    def __init__(self, o, x, csr, vocab, q, qs, live, P_max):
        self.o, self.vocab = o, vocab
        alive = bitmap(live) if not live.all() else None
        df, n_live, total = global_stats(csr, live, vocab)
        post = o.bm25_build(*live_csr(csr, live), vocab, df, n_live, total)
        self.dd, self.do = o.dense_topk(x, q, P_max, alive)
        self.bm = [o.bm25_query(post, t[t < vocab], P_max, alive) for t in qs]

    def check(self, got, k, P, vw, tw, mode, allow=None, hybrid=True, what=""):
        B = got["count"].shape[0]
        for b in range(B):
            dd, do = self.dd[b, :P], self.do[b, :P]
            if hybrid:
                bs, bo = self.bm[b][0][:P], self.bm[b][1][:P]
                keep = bo >= 0
                if allow is not None:
                    keep &= ((allow[np.maximum(bo, 0) >> 5] >> (np.maximum(bo, 0) & 31).astype(np.uint32)) & 1).astype(bool)
                fin, de, sp, rk, od = self.o.fuse(dd, do, bs[keep], bo[keep], k, vw, tw, mode)
            else:
                v = do >= 0
                od, de = do[v][:k], dd[v][:k]
                fin, sp, rk = de.astype(np.float64), np.full(len(od), np.nan, np.float32), np.full(len(od), -1, np.int32)
            c = len(od)
            w = (what, b)
            assert int(got["count"][b]) == c, w
            assert np.array_equal(got["ordinal"][b, :c], od), w
            assert np.array_equal(got["final"][b, :c], fin), w
            assert np.array_equal(got["rank"][b, :c], rk), w
            assert np.array_equal(got["dense"][b, :c], de, equal_nan=True), w
            assert np.array_equal(got["sparse"][b, :c], sp, equal_nan=True), w
            assert (got["ordinal"][b, c:] == -1).all() and (got["final"][b, c:] == 0.0).all(), w


def special_queries(csr, vocab, qs, rng):
    """0: the rarest term, matching fewer than P = 900 rows (the zero fill combines across shards); 1: no terms; 2: only
    out-of-vocabulary ids; 3: a duplicated term; 4: more than 32 terms"""
    off, ids, tf, dl = csr
    df = np.bincount(ids, minlength=vocab)
    rare = int(np.argmin(np.where(df > 0, df, np.iinfo(df.dtype).max)))
    assert df[rare] < 900                  # fewer matches than the pool at k = 300
    qs = list(qs)
    qs[0] = np.array([rare], np.uint32)
    qs[1] = np.zeros(0, np.uint32)
    qs[2] = np.array([vocab, vocab + 7, 0x7FFFFFFF], np.uint32)
    t = qs[3][0]
    qs[3] = np.array([t, qs[3][1] if len(qs[3]) > 1 else t, t], np.uint32)
    qs[4] = rng.integers(0, vocab, 40).astype(np.uint32)
    return qs


# ------------------------------------------------------------------------------------- service shapes, round robin
N_SVC, D_SVC, V_SVC, B_SVC = 600_001, 128, 30_000, 256   # 600,001: uneven shards at G = 2, 3 and 8


@pytest.fixture(scope="module")
def svc(oracle):
    from kaito_b200 import _native
    o = oracle
    x = o.synth_dense(N_SVC, D_SVC, 41)
    csr = o.synth_sparse(N_SVC, V_SVC, 42)
    q = o.synth_queries(x, B_SVC, 43)
    qs = special_queries(csr, V_SVC, o.synth_query_terms(V_SVC, B_SVC, 44, rank_offset=30), np.random.default_rng(45))
    ref = OracleRef(o, x, csr, V_SVC, q, qs, np.ones(N_SVC, bool), 900)
    ctx = _native.Context(0)
    single = ctx.create_index("svc_single", D_SVC)
    single.add(np.arange(N_SVC, dtype=np.uint64), x, *csr)
    single.commit(V_SVC)
    state = {"x": x, "csr": csr, "q": q, "qs": qs, "ref": ref, "ctx": ctx, "single": single, "shards": {}}
    yield state
    for sh in state["shards"].values():
        sh.drop()
    single.drop()
    ctx.close()


# (G, batch, k, K3 kernel, fusion mode, weights, allow): every value at least once; G = 2 with batches >= 16 (K2 on
# both shards), k = 300 with both K3 kernels and the zero-fill query, the allow bitmaps at G = 8
SVC_CASES = [
    (2, 256, 300, "warp", 0, (0.7, 0.3), None),
    (2, 16, 300, "legacy", 1, (0.5, 0.5), None),
    (2, 64, 10, "warp", 1, (0.7, 0.3), "vector"),
    (3, 15, 300, "warp", 0, (0.5, 0.5), None),
    (3, 1, 1, "legacy", 0, (0.7, 0.3), None),
    (3, 256, 10, "legacy", 1, (0.7, 0.3), None),
    (8, 64, 10, "legacy", 0, (0.7, 0.3), 0.03),
    (8, 16, 300, "warp", 1, (0.5, 0.5), 0.6),
    (8, 256, 1, "warp", 0, (0.7, 0.3), "vector"),
]


@pytest.mark.parametrize("G,batch,k,kernel,mode,weights,allow", SVC_CASES)
def test_round_robin_service_shapes(svc, loopback, monkeypatch, G, batch, k, kernel, mode, weights, allow):
    monkeypatch.setenv("KRAG_BM25_KERNEL", kernel)
    if G not in svc["shards"]:
        sh = Shards(loopback, svc["ctx"], f"svc_rr{G}", svc["x"], svc["csr"], V_SVC, G, "round_robin")
        n_docs, total, _ = zip(*sh.commit())
        assert set(n_docs) == {N_SVC} and set(total) == {int(svc["csr"][3].astype(np.int64).sum())}
        svc["shards"][G] = sh
    sh = svc["shards"][G]
    q, qs = svc["q"][:batch], svc["qs"][:batch]
    vw, tw = weights
    P = 3 * k
    if allow == "vector":
        got = sh.retrieve(q, None, k, vector_weight=vw, text_weight=tw, mode=mode)
        single = svc["single"].retrieve(q, None, k, vector_weight=vw, text_weight=tw, fusion_mode=mode)
        svc["ref"].check(got, k, P, vw, tw, mode, hybrid=False, what="vector-only")
        assert_same(got, single, "vector-only")
        return
    bm = None
    if allow is not None:
        bm = bitmap(np.random.default_rng(G * 100 + k).random(N_SVC) < allow)
    got = sh.retrieve(q, qs, k, vector_weight=vw, text_weight=tw, mode=mode, allow_bitmap=bm)
    single = svc["single"].retrieve(q, qs, k, vector_weight=vw, text_weight=tw, fusion_mode=mode, keyword_allow_bitmap=bm)
    svc["ref"].check(got, k, P, vw, tw, mode, allow=bm)
    assert_same(got, single, (G, batch, k))
    if bm is None:
        # the zero-fill query: its BM25 list is the rare term's rows, then the lowest global ordinals
        lst = sh.sr[0].last_lists[1, 0].cpu().numpy().view(np.uint64)
        bo = svc["ref"].bm[0][1][:P]
        assert np.array_equal((lst & M32).astype(np.int64), bo)


def test_empty_shards(oracle, loopback):
    """5 rows over 8 round-robin shards: shards 5, 6 and 7 hold no rows"""
    from kaito_b200 import _native
    o = oracle
    n, d, vocab = 5, 64, 50
    x = o.synth_dense(n, d, 51)
    csr = o.synth_sparse(n, vocab, 52, mean_len=12.0)
    q = o.synth_queries(x, 4, 53)
    qs = o.synth_query_terms(vocab, 4, 54, rank_offset=0)
    qs[1] = np.zeros(0, np.uint32)
    ctx = _native.Context(0)
    try:
        single = ctx.create_index("tiny_single", d)
        single.add(np.arange(n, dtype=np.uint64), x, *csr)
        single.commit(vocab)
        sh = Shards(loopback, ctx, "tiny_rr", x, csr, vocab, 8, "round_robin")
        try:
            sh.commit()
            ref = OracleRef(o, x, csr, vocab, q, qs, np.ones(n, bool), 30)
            for k, mode in ((10, 0), (1, 1)):
                got = sh.retrieve(q, qs, k, mode=mode)
                ref.check(got, k, 3 * k, 0.7, 0.3, mode, what=k)
                assert_same(got, single.retrieve(q, qs, k, fusion_mode=mode), k)
        finally:
            sh.drop()
            single.drop()
    finally:
        ctx.close()


# ------------------------------------------------------------------------------- tombstones and global statistics
def test_tombstones_and_recommits_under_global_statistics(oracle, loopback, monkeypatch):
    """Remove every row of shard 0 and a scattered 10 % elsewhere, commit (an incremental merge on the other shards,
    whose scores change because N, avgdl and df are global), then remove rows of one shard only and commit again.
    Each shard's postings must equal the oracle's build of its own rows under the global statistics."""
    from kaito_b200 import _native
    o = oracle
    n, d, vocab, G, k = 90_001, 64, 4000, 3, 300
    x = o.synth_dense(n, d, 61)
    csr = o.synth_sparse(n, vocab, 62)
    rng = np.random.default_rng(63)
    q = o.synth_queries(x, 20, 64)
    qs = special_queries(csr, vocab, o.synth_query_terms(vocab, 20, 65, rank_offset=20), rng)
    ctx = _native.Context(0)
    single = ctx.create_index("tomb_single", d)
    single.add(np.arange(n, dtype=np.uint64), x, *csr)
    single.commit(vocab)
    sh = Shards(loopback, ctx, "tomb_rr", x, csr, vocab, G, "round_robin")
    try:
        sh.commit()
        before = sh.ix[1].read_postings(int(qs[5][0]))
        live = np.ones(n, bool)
        dead = np.concatenate([np.arange(0, n, G), np.nonzero(rng.random(n) < 0.1)[0]])
        steps = [np.unique(dead), np.nonzero((np.arange(n) % G == 1) & (rng.random(n) < 0.2))[0]]
        for step, rm in enumerate(steps):
            rm = rm[live[rm]]
            live[rm] = False
            sh.remove(rm)
            single.remove(np.asarray(rm, np.uint64))
            sh.commit()
            assert _native.last_commit()["merged"] == 1           # an incremental merge, not a rebuild
            single.commit(vocab)
            df, n_live, total = global_stats(csr, live, vocab)
            for s in range(G):
                st = sh.ix[s].stats()
                assert (st.n_docs_global, st.total_len_global) == (n_live, total), s
                loc = live[sh.rows[s]]
                post = o.bm25_build(*live_csr(sub_csr(csr, sh.rows[s]), loc), vocab, df, n_live, total)
                terms = np.unique(np.concatenate([np.arange(12), rng.integers(0, vocab, 40), np.concatenate(qs[5:9])]))
                for t in terms:
                    docs, scores, cnt = sh.ix[s].read_postings(int(t), cap=len(sh.rows[s]) + 1)
                    sl = slice(post.off[t], post.off[t + 1])
                    assert cnt == post.off[t + 1] - post.off[t], (step, s, t)
                    assert np.array_equal(docs, post.doc[sl]) and np.array_equal(scores.view(np.uint32), post.score[sl].view(np.uint32)), (step, s, t)
            if step == 0:
                after = sh.ix[1].read_postings(int(qs[5][0]))
                assert not np.array_equal(after[1], before[1][np.isin(before[0], after[0])])   # global N moved every score
            ref = OracleRef(o, x, csr, vocab, q, qs, live, 3 * k)
            for kern in ("warp", "legacy"):
                monkeypatch.setenv("KRAG_BM25_KERNEL", kern)
                for kk, mode in ((k, 0), (10, 1)):
                    got = sh.retrieve(q, qs, kk, mode=mode)
                    ref.check(got, kk, 3 * kk, 0.7, 0.3, mode, what=(step, kern, kk))
                    assert_same(got, single.retrieve(q, qs, kk, fusion_mode=mode), (step, kern, kk))
    finally:
        sh.drop()
        single.drop()
        ctx.close()


# ------------------------------------------------------------------------------------- bench shape, contiguous
def _exact_bm25(ix, terms, vocab, n, P):
    """BM25 top-P recomputed in numpy from the index's postings: fp32 accumulation in query-term order (duplicates
    included, out-of-vocabulary ids skipped), (score desc, ordinal asc), zero-score rows fill by ascending ordinal"""
    acc = np.zeros(n, np.float32)
    for t in terms:
        if t >= vocab:
            continue
        docs, scores, cnt = ix.read_postings(int(t), cap=n + 1)
        assert cnt == len(docs)
        acc[docs.astype(np.int64)] += scores
    hit = np.nonzero(acc != 0)[0]
    keys = np.sort((((~_obits(acc[hit])) & M32) << np.uint64(32)) | hit.astype(np.uint64))[:P]
    ordn = (keys & M32).astype(np.int64)
    if len(ordn) < P:
        zeros = np.nonzero(acc == 0)[0][: P - len(ordn)]
        ordn = np.concatenate([ordn, zeros])
    return acc[ordn], ordn


def _obits(v):
    u = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & np.uint64(0x80000000), ~u & M32, u | np.uint64(0x80000000))


def test_bench_shape_contiguous_shards(oracle, loopback, monkeypatch):
    """3,000,000 x 256 rows (vocab 2^20), as one index and as 2 contiguous shards of 1.5M filled with row_base = lo:
    the same rows.  Under the default kernel choice the single index runs the warp K3 and the shards the legacy one,
    so (b) also cross-checks the two K3 generations at scale; 16 queries' BM25 lists are recomputed exactly in numpy."""
    from kaito_b200 import _native
    from kaito_b200.sharded import shard_range
    monkeypatch.delenv("KRAG_BM25_KERNEL", raising=False)
    n, d, vocab, G, B, seed = 3_000_000, 256, 1 << 20, 2, 256, 20260921
    ctx = _native.Context(0)
    single = ctx.create_index("bench_single", d)
    shards = []
    try:
        single.synth_fill(n, row_base=0, seed=seed, vocab=vocab)
        single.commit(vocab)
        from kaito_b200.sharded import NativeStages
        for s in range(G):
            lo, hi = shard_range(n, G, s)
            ix = ctx.create_index(f"bench_shard{s}", d)
            ix.synth_fill(hi - lo, row_base=lo, seed=seed, vocab=vocab)
            shards.append(ix)
        dpad = single.stats().dim_padded
        srs = [None] * G

        def mk(rank, group):
            srs[rank] = loopback.ShardedRetriever(NativeStages(ctx, shards[rank]), torch.device("cuda", 0), dpad, group=group)
            lo, hi = shard_range(n, G, rank)
            return srs[rank].commit(vocab, hi - lo)
        res = run_ranks(G, mk)
        assert [r[2] for r in res] == [0, n // 2]
        print(f"\nbench shape: the single index and its 2 shards hold {_native.device_bytes() / 2**30:.1f} GiB of device memory")
        s1 = single.stats()
        assert all((r[0], r[1]) == (s1.n_docs_global, s1.total_len_global) for r in res)
        rng = np.random.default_rng(71)
        rows = rng.integers(0, n, B // 2)
        q = np.concatenate([single.read_rows(int(r), 1) for r in rows])[:, :d]
        q = np.concatenate([q + 0.05 * rng.standard_normal(q.shape).astype(np.float32),
                            rng.standard_normal((B - len(rows), d)).astype(np.float32)])
        q = np.ascontiguousarray(q / np.linalg.norm(q, axis=1, keepdims=True), np.float32)
        qs = oracle.synth_query_terms(vocab, B, 72, rank_offset=100)
        qs[3] = np.array([vocab - 1], np.uint32)                   # rare: zero fill across the two shards
        for k in (10, 300):
            P = 3 * k

            def ret(rank, group):
                srs[rank].group = group
                out = srs[rank].retrieve(q, qs, k)
                return out, srs[rank].last_lists.cpu().numpy().view(np.uint64).copy()
            (got, lists), _ = run_ranks(G, ret)
            ref = single.retrieve(q, qs, k)
            assert_same(got, ref, k)
            sc, so = single.search_bm25(qs, P)
            for b in list(range(8)) + list(range(B - 8, B)):
                es, eo = _exact_bm25(single, qs[b], vocab, n, P)
                assert np.array_equal(so[b], eo) and np.array_equal(sc[b].view(np.uint32), es.view(np.uint32)), (k, b)
                assert np.array_equal((lists[1, b] & M32).astype(np.int64), eo), (k, b)
    finally:
        for ix in shards:
            ix.drop()
        single.drop()
        ctx.close()
