"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle on the
same seeded inputs.  Bit-exact for ids, ranks and fp32 scores (the kernels reproduce the
oracle's operation order); the north_star tolerance for dense scores is 1e-4."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "fuse_reference.json")


def _mk(ctx, name, dim):
    return ctx.create_index(name, dim)


@pytest.mark.parametrize("n,d,nq,P", [(1, 32, 1, 5), (63, 40, 2, 30), (1000, 384, 3, 30), (20000, 768, 5, 30),
                                      (5000, 1024, 4, 90), (4097, 100, 7, 900), (300, 768, 1, 900)])
def test_dense_scan_bit_exact(ctx_scan, oracle, n, d, nq, P):
    x = oracle.synth_dense(n, d, seed=n + d)
    q = oracle.synth_queries(x, nq, seed=n + d + 1)
    ix = _mk(ctx_scan, f"dense_{n}_{d}", d)
    try:
        ix.add(np.arange(n, dtype=np.uint64) + 1000, x)
        dist, ordn = ix.search_dense(q, P)
        rd, ro = oracle.dense_topk(x, q, P)
        assert np.array_equal(ordn, ro)
        assert np.array_equal(dist, rd)  # bit-exact, far inside the 1e-4 tolerance
        assert np.array_equal(ix.node_ids(ordn[ordn >= 0]), ordn[ordn >= 0].astype(np.uint64) + 1000)
    finally:
        ix.drop()


def test_dense_tombstones_and_appends(ctx_scan, oracle):
    x = oracle.synth_dense(3000, 128, seed=11)
    q = oracle.synth_queries(x, 4, seed=12)
    ix = _mk(ctx_scan, "tomb", 128)
    try:
        ix.add(np.arange(2000, dtype=np.uint64), x[:2000])
        ix.add(np.arange(2000, 3000, dtype=np.uint64), x[2000:])
        _, o0 = ix.search_dense(q, 10)
        dead = sorted(set(o0[:, :3].reshape(-1).tolist()))
        assert ix.remove(np.array(dead, np.uint64)) == len(dead)
        dist, ordn = ix.search_dense(q, 10)
        rd, ro = oracle.dense_topk(x, q, 10, oracle.alive_bitmap(3000, dead))
        assert np.array_equal(ordn, ro) and np.array_equal(dist, rd)
    finally:
        ix.drop()


@pytest.fixture(params=["warp", "legacy"])
def bm25_kernel(request, monkeypatch):
    """both generations of K3 on the small corpora (auto picks the first-generation kernel below 3M rows per shard)"""
    monkeypatch.setenv("KRAG_BM25_KERNEL", request.param)
    return request.param


def _sparse_index(ctx, oracle, n, vocab, d=32, seed=1):
    x = oracle.synth_dense(n, d, seed)
    off, ids, tf, dl = oracle.synth_sparse(n, vocab, seed + 1)
    ix = ctx.create_index(f"hyb_{n}_{vocab}", d)
    ix.add(np.arange(n, dtype=np.uint64), x, off, ids, tf, dl)
    ix.commit(vocab)
    return ix, x, (off, ids, tf, dl)


@pytest.mark.parametrize("n,vocab", [(50, 64), (3000, 2000), (40000, 30000)])
def test_bm25_postings_and_query_bit_exact(ctx_scan, oracle, n, vocab, bm25_kernel):
    ix, x, (off, ids, tf, dl) = _sparse_index(ctx_scan, oracle, n, vocab)
    try:
        post = oracle.bm25_build(off, ids, tf, dl, vocab)
        for t in list(range(0, min(vocab, 40))) + [vocab - 1]:
            docs, scores, cnt = ix.read_postings(t)
            sl = slice(post.off[t], post.off[t + 1])
            assert cnt == post.off[t + 1] - post.off[t]
            assert np.array_equal(docs, post.doc[sl]) and np.array_equal(scores, post.score[sl])
        qs = oracle.synth_query_terms(vocab, 9, seed=n, rank_offset=min(100, vocab // 8))
        qs[0] = np.concatenate([qs[0], qs[0][:2]])      # duplicated terms count twice
        qs[1] = np.array([vocab - 1], np.uint32)        # rare / empty posting list
        qs[2] = np.array([vocab + 5, 1], np.uint32)     # out-of-vocabulary id is ignored
        for P in (30, 90):
            score, ordn = ix.search_bm25(qs, P)
            for b, qt in enumerate(qs):
                rs, ro = oracle.bm25_query(post, qt[qt < vocab], P)
                assert np.array_equal(ordn[b], ro), (b, P)
                assert np.array_equal(score[b], rs)
    finally:
        ix.drop()


def test_bm25_long_queries_dense_postings(ctx_scan, oracle, bm25_kernel):
    """tiny vocabulary -> every term is frequent (thousands of postings per doc tile) and queries of
    40-70 terms span several term chunks and slab passes of the kernel's general path"""
    n, vocab = 40000, 48
    ix, x, (off, ids, tf, dl) = _sparse_index(ctx_scan, oracle, n, vocab)
    try:
        post = oracle.bm25_build(off, ids, tf, dl, vocab)
        g = np.random.default_rng(3)
        qs = [g.integers(0, vocab, m).astype(np.uint32) for m in (40, 70, 33, 1, 5)]
        for P in (30, 600):
            score, ordn = ix.search_bm25(qs, P)
            for b, qt in enumerate(qs):
                rs, ro = oracle.bm25_query(post, qt, P)
                assert np.array_equal(ordn[b], ro), (b, P)
                assert np.array_equal(score[b], rs)
    finally:
        ix.drop()


def test_bm25_zero_fill_and_tombstones(ctx_scan, oracle, bm25_kernel):
    ix, x, (off, ids, tf, dl) = _sparse_index(ctx_scan, oracle, 500, 800)
    try:
        post = oracle.bm25_build(off, ids, tf, dl, 800)
        rare = int(np.argmin(np.where(np.diff(post.off) > 0, np.diff(post.off), 1 << 30)))
        score, ordn = ix.search_bm25([np.array([rare], np.uint32)], 30)
        rs, ro = oracle.bm25_query(post, np.array([rare], np.uint32), 30)
        assert np.array_equal(ordn[0], ro) and np.array_equal(score[0], rs)
        assert (score[0] == 0).sum() > 0
        dead = ordn[0, :2].tolist() + [0, 1]
        ix.remove(np.array(sorted(set(dead)), np.uint64))
        score, ordn = ix.search_bm25([np.array([rare], np.uint32)], 30)
        rs, ro = oracle.bm25_query(post, np.array([rare], np.uint32), 30, oracle.alive_bitmap(500, dead))
        assert np.array_equal(ordn[0], ro) and np.array_equal(score[0], rs)
    finally:
        ix.drop()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [1, 777, 50_000])
def test_bm25_build_in_term_ranges(ctx_scan, oracle, monkeypatch, chunk, bm25_kernel):
    """the postings build sorts one TERM RANGE at a time (KRAG_BM25_BUILD_CHUNK postings per range; by default what fits in
    the free device memory): same postings, same tile index, same results -- also after tombstones and a re-commit"""
    monkeypatch.setenv("KRAG_BM25_BUILD_CHUNK", str(chunk))
    n, vocab = 40000, 3000
    ix, x, (off, ids, tf, dl) = _sparse_index(ctx_scan, oracle, n, vocab, seed=5)
    try:
        post = oracle.bm25_build(off, ids, tf, dl, vocab)
        for t in list(range(0, 60)) + list(range(vocab - 20, vocab)):
            docs, scores, cnt = ix.read_postings(t)
            sl = slice(post.off[t], post.off[t + 1])
            assert cnt == post.off[t + 1] - post.off[t]
            assert np.array_equal(docs, post.doc[sl]) and np.array_equal(scores, post.score[sl])
        qs = oracle.synth_query_terms(vocab, 12, seed=9, rank_offset=0)      # rank_offset 0: the most frequent terms (tile index rows)
        _bm25_batch_vs_oracle(ix, oracle, post, qs, (30, 200))
        dead = list(range(0, n, 7))
        ix.remove(np.array(dead, np.uint64))
        ix.commit(vocab)                                                      # rebuild without the tombstoned documents
        live = np.ones(n, bool); live[dead] = False
        keep = np.repeat(live, np.diff(off))
        off2 = np.concatenate([[0], np.cumsum(np.where(live, np.diff(off), 0))]).astype(np.int64)
        df = np.bincount(ids[keep], minlength=vocab).astype(np.uint32)
        post2 = oracle.bm25_build(off2, ids[keep], tf[keep], dl, vocab, df, int(live.sum()), int(dl[live].astype(np.int64).sum()))
        _bm25_batch_vs_oracle(ix, oracle, post2, qs, (30,), oracle.alive_bitmap(n, dead))
    finally:
        ix.drop()


def _bm25_batch_vs_oracle(ix, oracle, post, qs, pools, alive=None):
    for P in pools:
        score, ordn = ix.search_bm25(qs, P)
        for b, qt in enumerate(qs):
            rs, ro = oracle.bm25_query(post, qt[qt < post.off.size - 1], P, alive)
            assert np.array_equal(ordn[b], ro), (b, P)
            assert np.array_equal(score[b], rs), (b, P)


@pytest.fixture(scope="module")
def sparse_400k(ctx_scan, oracle):
    """400k documents: 98 sub-tiles of 4096 docs, frequent terms (tile index rows), mid terms (rows built per batch by
    bm25_resolve_kernel) and rare ones; two-pass path (sampled threshold, then the main pass)"""
    n, vocab = 400_000, 60_000
    ix, x, csr = _sparse_index(ctx_scan, oracle, n, vocab, d=32, seed=21)
    post = oracle.bm25_build(*csr, vocab)
    yield ix, post, n, vocab
    ix.drop()


def test_bm25_warp_kernel_two_pass_bit_exact(sparse_400k, oracle, monkeypatch):
    ix, post, n, vocab = sparse_400k
    monkeypatch.setenv("KRAG_BM25_KERNEL", "warp")               # auto would pick the first-generation kernel below 3M rows
    qs = oracle.synth_query_terms(vocab, 48, seed=5, rank_offset=20)
    qs[0] = np.concatenate([qs[0], qs[0]])                        # every term twice
    qs[1] = np.array([0, 1, 2, 3], np.uint32)                     # the most frequent terms: ~every document matches
    qs[2] = np.array([vocab - 1, vocab - 2, vocab + 9], np.uint32)
    g = np.random.default_rng(8)
    qs[3] = g.integers(0, 2000, 45).astype(np.uint32)             # > 32 terms: chunked accumulate-all-then-claim path
    _bm25_batch_vs_oracle(ix, oracle, post, qs, (30, 90, 900))


def test_bm25_overflow_takes_the_exact_safety_net(sparse_400k, oracle, monkeypatch):
    """a 64-entry candidate list overflows for every broad query: the overflow flag must route those queries through the
    legacy exact kernel, the others stay on the warp kernel; results identical"""
    ix, post, n, vocab = sparse_400k
    qs = oracle.synth_query_terms(vocab, 12, seed=6, rank_offset=20)
    qs[0] = np.array([vocab - 1], np.uint32)                      # a handful of matches: stays below the cap
    monkeypatch.setenv("KRAG_BM25_KERNEL", "warp")
    monkeypatch.setenv("KRAG_BM25_CAPQ", "64")
    _bm25_batch_vs_oracle(ix, oracle, post, qs, (30,))


def test_bm25_legacy_kernel_still_exact(sparse_400k, oracle, monkeypatch):
    """KRAG_BM25_KERNEL=legacy: the CTA-per-tile kernel alone (the safety net) on the 4096-doc tile index and 2048-posting short lists"""
    ix, post, n, vocab = sparse_400k
    qs = oracle.synth_query_terms(vocab, 10, seed=7, rank_offset=20)
    qs[1] = np.random.default_rng(9).integers(0, 3000, 40).astype(np.uint32)
    monkeypatch.setenv("KRAG_BM25_KERNEL", "legacy")
    _bm25_batch_vs_oracle(ix, oracle, post, qs, (30, 300))


@pytest.mark.parametrize("k", [1, 10, 40, 300])
def test_retrieve_matches_oracle_pipeline(ctx_scan, oracle, k, bm25_kernel):
    n, vocab, d = 6000, 5000, 64
    ix, x, (off, ids, tf, dl) = _sparse_index(ctx_scan, oracle, n, vocab, d=d, seed=7)
    try:
        post = oracle.bm25_build(off, ids, tf, dl, vocab)
        q = oracle.synth_queries(x, 6, seed=8)
        qs = oracle.synth_query_terms(vocab, 6, seed=9, rank_offset=50)
        P = oracle.pool_size(k)
        for mode in (0, 1):
            out = ix.retrieve(q, qs, k, fusion_mode=mode)
            for b in range(6):
                dd, do = oracle.dense_topk(x, q[b:b + 1], P)
                bs, bo = oracle.bm25_query(post, qs[b], P)
                fin, de, sp, rk, od = oracle.fuse(dd[0], do[0], bs, bo, k, mode=mode)
                c = out["count"][b]
                assert c == len(od)
                assert np.array_equal(out["ordinal"][b, :c], od)
                assert np.array_equal(out["final"][b, :c], fin)
                assert np.array_equal(out["rank"][b, :c], rk)
                assert np.array_equal(out["dense"][b, :c], de, equal_nan=True)
                assert np.array_equal(out["sparse"][b, :c], sp, equal_nan=True)
        # vector-only fallback (hybrid_retriever.py:216-218)
        out = ix.retrieve(q, None, k)
        dd, do = oracle.dense_topk(x, q, P)
        kk = min(k, P)
        assert np.array_equal(out["ordinal"][:, :kk], do[:, :kk])
        # keyword-side metadata post-filter: only even rows allowed
        allow = np.zeros((n + 31) // 32, np.uint32)
        ev = np.arange(0, n, 2)
        np.bitwise_or.at(allow, ev >> 5, np.uint32(1) << (ev & 31).astype(np.uint32))
        out = ix.retrieve(q[:2], qs[:2], k, keyword_allow_bitmap=allow)
        for b in range(2):
            dd, do = oracle.dense_topk(x, q[b:b + 1], P)
            bs, bo = oracle.bm25_query(post, qs[b], P)
            keep = (bo % 2 == 0) & (bo >= 0)
            fin, de, sp, rk, od = oracle.fuse(dd[0], do[0], bs[keep], bo[keep], k)
            c = out["count"][b]
            assert np.array_equal(out["ordinal"][b, :c], od) and np.array_equal(out["final"][b, :c], fin)
    finally:
        ix.drop()


def test_fuse_kernel_against_reference_golden(ctx_scan):
    """golden lists produced by the reference's own _fuse go through the CUDA fuse kernel"""
    import torch
    from kaito_b200 import _native
    gold = json.load(open(GOLD))

    def okey(v, asc=True):
        u = np.float32(v).view(np.uint32).astype(np.uint64)
        o = np.where(u & np.uint64(0x80000000), ~u & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))
        return o if asc else (~o & np.uint64(0xFFFFFFFF))

    for c in gold["fuse"]:
        k = c["k"]
        P = max(len(c["dense_ids"]), len(c["bm25_ids"]), 1)
        dk = np.full(P, _native.KRAG_KEY_PAD, np.uint64)
        bk = np.full(P, _native.KRAG_KEY_PAD, np.uint64)
        if c["dense_ids"]:
            dk[: len(c["dense_ids"])] = (okey(np.array(c["dense_dist"], np.float32)) << np.uint64(32)) | np.array(c["dense_ids"], np.uint64)
        if c["bm25_ids"]:
            bk[: len(c["bm25_ids"])] = (okey(np.array(c["bm25_score"], np.float32), False) << np.uint64(32)) | np.array(c["bm25_ids"], np.uint64)
        t = lambda a: torch.from_numpy(a.view(np.int64)).cuda()
        d_dk, d_bk = t(dk), t(bk)
        fin = torch.empty(k, dtype=torch.float64, device="cuda")
        de = torch.empty(k, dtype=torch.float32, device="cuda")
        sp = torch.empty(k, dtype=torch.float32, device="cuda")
        rk = torch.empty(k, dtype=torch.int32, device="cuda")
        od = torch.empty(k, dtype=torch.int64, device="cuda")
        cnt = torch.empty(1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx_scan.dev_fuse(1, P, k, d_dk.data_ptr(), d_bk.data_ptr(), c["vector_weight"], c["text_weight"], 0, None,
                          fin.data_ptr(), de.data_ptr(), sp.data_ptr(), rk.data_ptr(), od.data_ptr(), cnt.data_ptr(), 0)
        torch.cuda.synchronize()
        n = int(cnt.item())
        assert n == len(c["out_ids"])
        assert fin[:n].cpu().tolist() == c["out_final"]          # fp64 bit-exact with the reference
        got, ref = od[:n].cpu().tolist(), c["out_ids"]
        f = c["out_final"]
        i = 0
        while i < n:                                             # ids equal up to the reference's unspecified tie order
            j = i
            while j < n and f[j] == f[i]:
                j += 1
            if j < n or len(set(f)) == len(f):
                assert sorted(got[i:j]) == sorted(ref[i:j])
            i = j


def test_persist_load_roundtrip(ctx_scan, oracle, tmp_path):
    ix, x, (off, ids, tf, dl) = _sparse_index(ctx_scan, oracle, 700, 900, d=48, seed=21)
    try:
        ix.remove(np.array([5, 6], np.uint64))
        q = oracle.synth_queries(x, 2, seed=22)
        qs = oracle.synth_query_terms(900, 2, seed=23, rank_offset=10)
        ix.commit(900)
        a = ix.retrieve(q, qs, 10)
        ix.persist(str(tmp_path / "snap"))
        ix2 = ctx_scan.load_index("reloaded", str(tmp_path / "snap"))
        try:
            b = ix2.retrieve(q, qs, 10)
            for key in a:
                assert np.array_equal(a[key], b[key], equal_nan=True), key
        finally:
            ix2.drop()
    finally:
        ix.drop()


def test_full_size_properties(ctx_scan, oracle):
    """size-independent checks at a size the oracle cannot brute-force in seconds:
    device-generated 2M x 768 corpus; returned distances are re-derived on the CPU from the
    rows read back; a planted query returns its row first; batched == single-query results."""
    n, d = 2_000_000, 768
    ix = ctx_scan.create_index("big", d)
    try:
        ix.synth_fill(n, row_base=0, seed=5)
        rows = np.array([3, 999_999, 1_999_999])
        xr = np.concatenate([ix.read_rows(int(r), 1) for r in rows])
        assert np.allclose(np.linalg.norm(xr, axis=1), 1.0, atol=1e-5)
        q = xr + 0.01 * oracle.synth_dense(3, d, 1)
        dist, ordn = ix.search_dense(q, 10)
        assert ordn[:, 0].tolist() == rows.tolist()
        assert (np.diff(dist, axis=1) >= 0).all()
        for b in range(3):
            got_rows = np.concatenate([ix.read_rows(int(o), 1) for o in ordn[b]])
            assert np.array_equal(oracle.l2sq(got_rows, q[b]), dist[b])
            # a random sample of other rows never beats the k-th distance
            samp = np.random.default_rng(b).integers(0, n, 64)
            sd = oracle.l2sq(np.concatenate([ix.read_rows(int(r), 1) for r in samp]), q[b])
            assert ((sd >= dist[b, -1]) | np.isin(samp, ordn[b])).all()
        d1, o1 = ix.search_dense(q[:1], 10)
        assert np.array_equal(o1[0], ordn[0]) and np.array_equal(d1[0], dist[0])
    finally:
        ix.drop()


@pytest.mark.gpu
def test_peer_exchange_single_rank_roundtrip(ctx_scan):
    """krag_p2p with world = 1: push into the own mailbox + flag-waiting merge must return the sorted lists unchanged,
    across repeated exchanges (parity slots) and changing shapes. The world > 1 case is covered on a 2-GPU box by
    scripts/sharded_gpu_check.py (peer-memory path == NCCL path == single-shard oracle)."""
    import torch
    from kaito_b200 import _native
    p = _native.P2PExchange(ctx_scan, 0, 1, 64, 64)
    p.connect(p.handle.copy())
    rng = np.random.default_rng(5)
    for it, (nl, B, P) in enumerate([(2, 7, 30), (1, 64, 64), (2, 1, 3), (2, 64, 64), (1, 5, 17)]):
        keys = np.sort(rng.integers(0, 2**62, size=(nl, B, P), dtype=np.uint64), axis=-1)
        keys[0, 0, P - 1] = np.uint64(2**64 - 1)      # a padded (short) list stays padded
        d_in = torch.from_numpy(keys.view(np.int64)).cuda()
        d_out = torch.empty_like(d_in)
        p.exchange_merge(nl, B, P, d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert np.array_equal(d_out.cpu().numpy().view(np.uint64), keys), it
    with pytest.raises(_native.KragError):
        p.exchange_merge(2, 64, 65, d_in.data_ptr(), d_out.data_ptr(), 0)   # larger than the agreed mailbox
    p.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("dense_mode,batch", [(1, 3), (0, 40)])
def test_filter_pushdown_bit_exact(oracle, dense_mode, batch):
    """KRAG_FILTER_PUSHDOWN: the allow bitmap (AND tombstones) is honoured inside K1 / K2 / K3 -- compared with the
    oracle run on eligible = allow & alive for both lists (ids and fused scores bit-exact); 3% and 60% selectivity."""
    from kaito_b200 import _native
    o = oracle
    n, d, vocab, k = 300_000 if dense_mode == 0 else 60_000, 128, 5000, 10
    x = o.synth_dense(n, d, 21)
    off, ids, tf, dl = o.synth_sparse(n, vocab, 22)
    q = o.synth_queries(x, batch, 23)
    qs = o.synth_query_terms(vocab, batch, 24, rank_offset=30)
    c = _native.Context(0, dense_mode=dense_mode)
    try:
        ix = c.create_index("pd", d)
        ix.add(np.arange(n, dtype=np.uint64), x, off, ids, tf, dl)
        dead = set(range(0, n, 7))
        ix.remove(np.array(sorted(dead), np.uint64))
        ix.commit(vocab)
        live = np.ones(n, bool); live[list(dead)] = False
        keep = np.repeat(live, np.diff(off))
        off2 = np.concatenate([[0], np.cumsum(np.where(live, np.diff(off), 0))]).astype(np.int64)
        df = np.bincount(ids[keep], minlength=vocab).astype(np.uint32)
        post = o.bm25_build(off2, ids[keep], tf[keep], dl, vocab, df, int(live.sum()), int(dl[live].astype(np.int64).sum()))
        alive = o.alive_bitmap(n, dead)
        rng = np.random.default_rng(9)
        P = o.pool_size(k)
        for frac in (0.03, 0.6):
            allow = np.packbits(rng.random(((n + 31) // 32) * 32) < frac, bitorder="little").view(np.uint32)
            got = ix.retrieve(q, qs, k, fusion_mode=_native.FILTER_PUSHDOWN, keyword_allow_bitmap=allow)
            got_v = ix.retrieve(q, None, k, fusion_mode=_native.FILTER_PUSHDOWN, keyword_allow_bitmap=allow)
            elig = allow & alive
            for b in range(batch):
                dd, do = o.dense_topk(x, q[b:b + 1], P, elig)
                bs, bo = o.bm25_query(post, qs[b], P, elig)
                fin, de, sp, rk, od = o.fuse(dd[0], do[0], bs, bo, k)
                cnt = int(got["count"][b])
                assert cnt == len(od) and np.array_equal(got["ordinal"][b, :cnt], od), (frac, b)
                assert np.array_equal(got["final"][b, :cnt], fin)
                assert all((elig[o_ >> 5] >> (o_ & 31)) & 1 for o_ in got["ordinal"][b, :cnt])
                assert np.array_equal(got_v["ordinal"][b, :k], do[0, :k]) and np.array_equal(got_v["final"][b, :k], dd[0, :k].astype(np.float64))
        ix.drop()
    finally:
        c.close()


@pytest.mark.parametrize("kernel", ["warp", "legacy"])
def test_strided_ordinal_map(ctx_scan, oracle, monkeypatch, kernel):
    """round-robin shards of the multi-GPU service: global ordinal = base + row * stride in every kernel that builds keys
    (K1, K2 rescoring, K3 claim, zero fill) and back again in krag_index_node_ids"""
    monkeypatch.setenv("KRAG_BM25_KERNEL", kernel)
    n, vocab, d, base, stride = 300_000, 3000, 64, 3, 5
    x = oracle.synth_dense(n, d, 31)
    off, ids, tf, dl = oracle.synth_sparse(n, vocab, 32)
    ix = ctx_scan.create_index("strided", d)
    try:
        ix.add(np.arange(n, dtype=np.uint64) + 7, x, off, ids, tf, dl)
        ix.set_ordinal_map(base, stride)
        ix.commit(vocab)
        assert ix.stats().ordinal_base == base
        q = oracle.synth_queries(x, 20, 33)
        for qq in (q[:3], q):                                   # K1 (batch < 16) and K2 (prune + exact rescoring)
            dist, ordn = ix.search_dense(qq, 30)
            rd, ro = oracle.dense_topk(x, qq, 30)
            assert np.array_equal(ordn, base + stride * ro) and np.array_equal(dist, rd)
        post = oracle.bm25_build(off, ids, tf, dl, vocab)
        qs = oracle.synth_query_terms(vocab, 6, seed=34, rank_offset=30)
        qs[0] = np.array([vocab - 1], np.uint32)                # short list -> zero-score fill
        score, ordn = ix.search_bm25(qs, 30)
        for b, qt in enumerate(qs):
            rs, ro = oracle.bm25_query(post, qt, 30)
            assert np.array_equal(ordn[b], np.where(ro >= 0, base + stride * ro, -1)) and np.array_equal(score[b], rs)
        assert np.array_equal(ix.node_ids(ordn[1]), (ordn[1] - base) // stride + 7)
        with pytest.raises(Exception):
            ix.node_ids(np.array([base + 1], np.int64))          # not a multiple of the stride: not this shard's
    finally:
        ix.drop()
