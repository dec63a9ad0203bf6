"""krag_index_compact on the H100: a compacted index answers exactly as a fresh index built from its live rows in the same
order (every dense mode, both row storages, removal patterns that stress the in-place window schedule), results are unchanged
across a compaction with stale statistics, and the memory of the removed rows is returned."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_ROWS, DIM, VOCAB = 262144, 768, 30000
W_X = (32 << 20) // (DIM * 4)           # rows per staging window of the fp32 rows (COMPACT_STAGE_BYTES)


@pytest.fixture(scope="module")
def N():
    from kaito_b200 import _native
    return _native


@pytest.fixture(scope="module")
def corpus(oracle):
    x = oracle.synth_dense(N_ROWS, DIM, 31)
    off, tid, tf, dl = oracle.synth_sparse(N_ROWS, VOCAB, 32, mean_len=24.0)
    q = oracle.synth_queries(x, 256, 33)
    qt = oracle.synth_query_terms(VOCAB, 256, 34, rank_offset=20)
    return x, off, tid, tf, dl, q, qt


@pytest.fixture(scope="module")
def contexts(N):
    # the device context keeps a bf16 shadow of the rows (DENSE_TC_BF16 at creation), so compaction moves it too
    dev = N.Context(device_id=0, dense_mode=N.DENSE_TC_BF16)
    host = N.Context(device_id=0, row_storage=N.ROWS_HOST)
    yield {"device": dev, "host": host}
    dev.close()
    host.close()


def _patterns():
    n, rng = N_ROWS, np.random.default_rng(35)
    pats = {"none": np.ones(n, bool), "all": np.zeros(n, bool)}
    a = np.ones(n, bool); a[0] = False; pats["row0"] = a
    a = np.ones(n, bool); a[-1000:] = False; pats["last"] = a
    pats["every_other"] = np.arange(n) % 2 == 1
    a = np.ones(n, bool)
    for s in (30, W_X - 3, 2 * W_X - 40, 2 * (W_X * 2) - 5, 5 * W_X + 31):   # across bitmap words and staging windows
        a[s:s + 45] = False
    pats["runs"] = a
    pats["random30"] = rng.random(n) >= 0.3
    return pats


def _subset(corpus, live):
    x, off, tid, tf, dl = corpus[:5]
    rows = np.flatnonzero(live)
    lens = np.diff(off)[rows]
    keep = np.repeat(live, np.diff(off))
    return rows, x[rows], np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), tid[keep], tf[keep], dl[rows]


def _build(ctx, name, ids, x, off, tid, tf, dl):
    ix = ctx.create_index(name, DIM)
    if len(ids):
        ix.add(ids, x, off, tid, tf, dl)
    return ix


def _allow(ids):
    """keyword bitmap over rows: node id % 3 != 0"""
    bits = (np.asarray(ids, np.int64) % 3 != 0)
    bm = np.zeros(max(1, (len(bits) + 31) // 32), np.uint32)
    for r in np.flatnonzero(bits):
        bm[r >> 5] |= np.uint32(1 << (r & 31))
    return bm


def _outcome(f):
    from kaito_b200._native import KragError
    try:
        return f()
    except KragError as e:
        return ("error", e.code)


def _searches(N, ix, q, qt, bm, dense_modes):
    out = {}
    for mode in dense_modes:
        ix.set_dense_mode(mode)
        for P in (1, 30, 900):
            for B in (1, 16, 256):
                out[("dense", mode, P, B)] = _outcome(lambda: ix.search_dense(q[:B], P))
    for P in (1, 30, 900):
        for B in (1, 16, 256):
            out[("bm25", P, B)] = _outcome(lambda: ix.search_bm25(qt[:B], P))
    for flt, mode in ((None, 0), ("post", 0), ("push", N.FILTER_PUSHDOWN)):
        r = _outcome(lambda: ix.retrieve(q[:64], qt[:64], 10, keyword_allow_bitmap=bm if flt else None, fusion_mode=mode))
        if isinstance(r, dict):
            r = [(c, r["ordinal"][b, :c].copy(), r["final"][b, :c].copy(), r["dense"][b, :c].copy(), r["sparse"][b, :c].copy())
                 for b, c in enumerate(r["count"])]
        out[("retrieve", flt)] = r
    return out


def _same(a, b):
    if isinstance(a, tuple) and a and isinstance(a[0], str):
        return a == b
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def _assert_same(ra, rb):
    assert ra.keys() == rb.keys()
    bad = [k for k in ra if not _same(ra[k], rb[k])]
    assert not bad, f"differ: {bad[:5]}"


STAT_FIELDS = ("n_rows", "n_live", "nnz", "n_docs_global", "total_len_global", "vocab", "ordinal_base", "dim", "dim_padded",
               "committed")


def _stats(ix):
    s = ix.stats()
    return {f: getattr(s, f) for f in STAT_FIELDS}


def _modes(N, storage):
    m = [N.DENSE_AUTO, N.DENSE_SCAN, N.DENSE_TC, N.DENSE_TC_BF16]
    return m + [N.DENSE_TC_TF32] if storage == "device" else m


def _compare_with_fresh(N, ctx, storage, A, B, live_ids, corpus):
    q, qt = corpus[5], corpus[6]
    assert _stats(A) == _stats(B)
    n = int(live_ids.size)
    if n:
        for r0 in range(0, n, 65536):
            m = min(65536, n - r0)
            assert np.array_equal(A.read_rows(r0, m), B.read_rows(r0, m))
    terms = np.unique(np.concatenate([np.arange(64), np.random.default_rng(36).integers(0, VOCAB, 136)]))
    for t in terms:
        da, sa, ca = A.read_postings(int(t), cap=n + 1)
        db, sb, cb = B.read_postings(int(t), cap=n + 1)
        assert ca == cb and np.array_equal(da, db) and np.array_equal(sa, sb), t
    if storage == "device" and n:
        assert np.array_equal(A.debug_tc_dump(q[:64]), B.debug_tc_dump(q[:64]))
    bm = _allow(live_ids)
    _assert_same(_searches(N, A, q, qt, bm, _modes(N, storage)), _searches(N, B, q, qt, bm, _modes(N, storage)))
    A.set_dense_mode(N.DENSE_TC_BF16 if storage == "device" else N.DENSE_AUTO)


@pytest.mark.parametrize("storage", ["device", "host"])
@pytest.mark.parametrize("pattern", list(_patterns()))
def test_compacted_index_equals_fresh_build(N, corpus, contexts, storage, pattern, tmp_path):
    ctx = contexts[storage]
    live = _patterns()[pattern]
    ids = np.arange(N_ROWS, dtype=np.uint64) + 1000
    x, off, tid, tf, dl = corpus[:5]
    A = _build(ctx, "A", ids, x, off, tid, tf, dl)
    B = None
    try:
        dead = ids[~live]
        assert A.remove(dead) == dead.size
        A.commit(VOCAB)
        bytes_before = A.stats().device_bytes
        assert A.compact() == dead.size
        if pattern == "none":
            assert A.stats().device_bytes == bytes_before
        else:
            assert A.stats().device_bytes < bytes_before
        rows, xs, offs, tids, tfs, dls = _subset(corpus, live)
        if pattern == "all":
            # an empty index that still takes adds and commits: then equal to a fresh build of the new rows
            assert A.stats().n_rows == 0 and A.stats().committed
            dA, oA = A.search_dense(corpus[5][:16], 30)
            assert (oA == -1).all() and np.isinf(dA).all()
            rows = np.arange(2000)
            xs, offs, tids, tfs, dls = x[:2000], off[:2001], tid[:off[2000]], tf[:off[2000]], dl[:2000]
            A.add(ids[rows], xs, offs, tids, tfs, dls)
            A.commit(VOCAB)
        B = _build(ctx, "B", ids[rows], xs, offs, tids, tfs, dls)
        B.commit(VOCAB)
        _compare_with_fresh(N, ctx, storage, A, B, ids[rows], corpus)
        if pattern == "random30":
            # after a compaction: adds, a remove by node id and a persist / load round trip
            g = np.random.default_rng(37)
            new_ids = np.arange(500, dtype=np.uint64) + 10_000_000
            nx = g.standard_normal((500, DIM), dtype=np.float32)
            sub = slice(0, 501)
            for ix in (A, B):
                ix.add(new_ids, nx, off[sub] - off[0], tid[off[0]:off[500]], tf[off[0]:off[500]], dl[:500])
                assert ix.remove(np.concatenate([ids[rows[[3, 7, 100]]], new_ids[[9]]])) == 4
                ix.commit(VOCAB)
            live_ids = np.concatenate([np.delete(ids[rows], [3, 7, 100]), np.delete(new_ids, [9])])
            bm = _allow(np.concatenate([ids[rows], new_ids]))
            _assert_same(_searches(N, A, corpus[5], corpus[6], bm, [N.DENSE_AUTO]), _searches(N, B, corpus[5], corpus[6], bm, [N.DENSE_AUTO]))
            assert A.compact() == 4 and B.compact() == 4
            _compare_with_fresh(N, ctx, storage, A, B, live_ids, corpus)
            A.persist(str(tmp_path))
            C = ctx.load_index("C", str(tmp_path))
            try:
                _compare_with_fresh(N, ctx, storage, A, C, live_ids, corpus)
            finally:
                C.drop()
    finally:
        A.drop()
        if B is not None:
            B.drop()


def _mapped(ix, out):
    res = []
    for b, c in enumerate(out["count"]):
        o = out["ordinal"][b, :c]
        res.append((ix.node_ids(o).tolist() if c else [], out["final"][b, :c].tolist()))
    return res


@pytest.mark.parametrize("storage", ["device", "host"])
def test_removed_since_last_commit_and_uncommitted(N, corpus, contexts, storage):
    ctx = contexts[storage]
    live = _patterns()["random30"]
    ids = np.arange(N_ROWS, dtype=np.uint64) + 7
    x, off, tid, tf, dl, q, qt = corpus
    rows, xs, offs, tids, tfs, dls = _subset(corpus, live)
    A = _build(ctx, "A", ids, x, off, tid, tf, dl)
    B = _build(ctx, "B", ids[rows], xs, offs, tids, tfs, dls)
    U = _build(ctx, "U", ids, x, off, tid, tf, dl)
    try:
        # removed since the last commit: the postings still hold the removed rows and the statistics are stale
        A.commit(VOCAB)
        A.remove(ids[~live])
        before = {}
        for mode in _modes(N, storage):
            A.set_dense_mode(mode)
            d, o = A.search_dense(q, 30)
            before[mode] = (d, A.node_ids(np.where(o >= 0, o, 0)), o >= 0)
        sb = A.search_bm25(qt, 30)
        sb_ids = A.node_ids(np.maximum(sb[1], 0))
        r_before = _mapped(A, A.retrieve(q[:64], qt[:64], 10))
        s_before = _stats(A)
        assert A.compact() == int((~live).sum())
        for mode in _modes(N, storage):
            A.set_dense_mode(mode)
            d, o = A.search_dense(q, 30)
            assert np.array_equal(d, before[mode][0]) and np.array_equal(o >= 0, before[mode][2])
            assert np.array_equal(np.where(o >= 0, A.node_ids(np.where(o >= 0, o, 0)), 0), np.where(before[mode][2], before[mode][1], 0))
        sa = A.search_bm25(qt, 30)
        assert np.array_equal(sa[0], sb[0]) and np.array_equal(sa[1] >= 0, sb[1] >= 0)
        assert np.array_equal(A.node_ids(np.maximum(sa[1], 0))[sa[1] >= 0], sb_ids[sb[1] >= 0])
        assert r_before == _mapped(A, A.retrieve(q[:64], qt[:64], 10))
        s_after = _stats(A)
        assert s_after["n_docs_global"] == s_before["n_docs_global"] and s_after["total_len_global"] == s_before["total_len_global"]
        # the next commit: a fresh build
        A.commit(VOCAB)
        B.commit(VOCAB)
        _compare_with_fresh(N, ctx, storage, A, B, ids[rows], corpus)
        # never committed: add, remove, compact, commit
        U.remove(ids[~live])
        assert U.compact() == int((~live).sum()) and not U.stats().committed
        U.commit(VOCAB)
        _compare_with_fresh(N, ctx, storage, U, B, ids[rows], corpus)
    finally:
        for ix in (A, B, U):
            ix.drop()


@pytest.mark.parametrize("storage", ["device", "host"])
def test_large_index_returns_its_memory(N, storage):
    n, dim, vocab = 3_200_000, 256, 1 << 16
    ctx = N.Context(device_id=0, row_storage=N.ROWS_HOST if storage == "host" else N.ROWS_DEVICE)
    try:
        ix = ctx.create_index("big", dim)
        ix.synth_fill(n, 0, 41, vocab)
        raw_nnz = ix.stats().nnz
        g = np.random.default_rng(42)
        dead = np.flatnonzero(g.random(n) < 0.5).astype(np.uint64)
        assert ix.remove(dead) == dead.size
        ix.commit(vocab)
        q = g.standard_normal((64, dim), dtype=np.float32)
        qt = [g.integers(0, vocab, 6).astype(np.uint32) for _ in range(64)]
        before = _mapped(ix, ix.retrieve(q, qt, 10))
        s0, dev0, pin0 = ix.stats(), N.device_bytes(), N.host_pinned_bytes()
        assert ix.compact() == dead.size
        s1, dev1, pin1 = ix.stats(), N.device_bytes(), N.host_pinned_bytes()
        assert s1.n_rows == n - dead.size and s1.n_live == s1.n_rows
        assert before == _mapped(ix, ix.retrieve(q, qt, 10))
        dpad = s1.dim_padded
        removed_entries = raw_nnz - s1.nnz           # s1.nnz: postings of a committed index = every entry of the live rows
        per_row = (2 * dpad + 4 + 4 if storage == "host" else 4 * dpad + 4) + 4 + 8     # rows, xnorm (+ xres), dlen, toff
        expect = dead.size * per_row + removed_entries * 6
        assert s0.device_bytes - s1.device_bytes >= 0.9 * expect
        assert dev0 - dev1 >= 0.9 * expect
        if storage == "host":
            assert pin0 - pin1 >= 0.9 * dead.size * 4 * dpad
        ix.drop()
    finally:
        ctx.close()


def test_round_robin_shard_is_refused(N, corpus, contexts):
    ctx = contexts["device"]
    x, off, tid, tf, dl, q, qt = corpus
    n = 5000
    ids = np.arange(n, dtype=np.uint64)
    ix = _build(ctx, "rr", ids, x[:n], off[:n + 1], tid[:off[n]], tf[:off[n]], dl[:n])
    try:
        ix.remove(ids[::3])
        ix.set_ordinal_map(0, 2)
        ix.commit(VOCAB)
        s0, r0 = _stats(ix), ix.search_dense(q[:16], 30)
        with pytest.raises(N.KragError) as e:
            ix.compact()
        assert e.value.code == N.KRAG_E_UNSUPPORTED
        assert _stats(ix) == s0
        r1 = ix.search_dense(q[:16], 30)
        assert np.array_equal(r0[0], r1[0]) and np.array_equal(r0[1], r1[1])
    finally:
        ix.drop()
