"""Incremental BM25 commit on the H100: after any history of adds, removes, commits and compactions, the merged postings of an
index equal, bit for bit, a full build of the same rows.  The reference is a twin: a fresh index that replays the same adds
and removes (same node ids, same order) and commits once, so its commit is a full build."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIM = 64
RARE_MAX, SUB_DOCS = 2048, 2048


@pytest.fixture(scope="module")
def N():
    from kaito_b200 import _native
    return _native


@pytest.fixture(scope="module")
def ctx(N):
    c = N.Context(device_id=0)
    yield c
    c.close()


def rows(rng, n, vocab, mean_len=12, extra=None, empty_every=0):
    """n rows: vectors, CSR term lists (unique ids, Zipf-like), tf, doc_len.  extra: term id added to every row."""
    x = rng.standard_normal((n, DIM), dtype=np.float32)
    lens = np.minimum(rng.poisson(mean_len, n) + 1, vocab)
    if empty_every:
        lens[::empty_every] = 0
    ids, off = [], [0]
    for i in range(n):
        t = np.unique((rng.zipf(1.2, lens[i]) - 1) % vocab).astype(np.uint32)
        if extra is not None:
            t = np.unique(np.append(t, np.uint32(extra)))
        ids.append(t)
        off.append(off[-1] + t.size)
    tid = np.concatenate(ids) if off[-1] else np.zeros(0, np.uint32)
    tf = rng.integers(1, 6, tid.size).astype(np.uint16)
    dl = np.array([int(tf[off[i]:off[i + 1]].sum()) + int(rng.integers(0, 8)) for i in range(n)], np.uint32)
    return x, np.array(off, np.int64), tid, tf, dl


class History:
    """an index that commits whenever asked, and the log that builds its twin"""

    def __init__(self, ctx, name):
        self.ctx, self.name, self.log, self.next_id = ctx, name, [], 1
        self.ix = ctx.create_index(name, DIM)

    def add(self, data, ids=None):
        n = data[0].shape[0]
        if ids is None:
            ids = np.arange(self.next_id, self.next_id + n, dtype=np.uint64)
            self.next_id += n
        self.ix.add(ids, *data)
        self.log.append(("add", ids, data))
        return ids

    def remove(self, ids):
        self.log.append(("remove", np.asarray(ids, np.uint64)))
        return self.ix.remove(ids)

    def twin(self, vocab, ctx=None):
        t = (ctx or self.ctx).create_index(self.name + "_twin", DIM)
        for op in self.log:
            if op[0] == "add":
                t.add(op[1], *op[2])
            else:
                t.remove(op[1])
        t.commit(vocab)
        return t


def queries(rng, vocab, n=64):
    q = rng.standard_normal((n, DIM), dtype=np.float32)
    qt = [np.unique((rng.zipf(1.3, int(rng.integers(1, 6))) - 1) % vocab).astype(np.uint32) for _ in range(n)]
    return q, qt


def same_arrays(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def assert_same_index(A, B, vocab, terms=None, device_bytes=True, seed=0):
    sa, sb = A.stats(), B.stats()
    assert sa.committed and sb.committed
    for f in ("nnz", "n_docs_global", "total_len_global", "n_rows", "n_live", "vocab"):
        assert getattr(sa, f) == getattr(sb, f), f
    if device_bytes:
        assert sa.device_bytes == sb.device_bytes
    cap = sa.n_rows + 1
    for t in (range(vocab) if terms is None else terms):
        da, xa, ca = A.read_postings(int(t), cap=cap)
        db, xb, cb = B.read_postings(int(t), cap=cap)
        assert ca == cb and np.array_equal(da, db) and np.array_equal(xa.view(np.uint32), xb.view(np.uint32)), t
    rng = np.random.default_rng(seed)
    q, qt = queries(rng, vocab)
    old = os.environ.get("KRAG_BM25_KERNEL")
    try:
        for kern in ("warp", "legacy"):
            os.environ["KRAG_BM25_KERNEL"] = kern
            for P in (1, 30, 300):
                ra, rb = A.search_bm25(qt, P), B.search_bm25(qt, P)
                assert same_arrays(ra[0], rb[0]) and same_arrays(ra[1], rb[1]), (kern, P)
    finally:
        if old is None:
            os.environ.pop("KRAG_BM25_KERNEL", None)
        else:
            os.environ["KRAG_BM25_KERNEL"] = old
    ra, rb = A.retrieve(q, qt, 10), B.retrieve(q, qt, 10)
    for k in ra:
        assert same_arrays(ra[k], rb[k]), k


def checkpoint(h, vocab, **kw):
    h.ix.commit(vocab)
    T = h.twin(vocab)
    try:
        assert_same_index(h.ix, T, vocab, **kw)
    finally:
        T.drop()


def test_adds_growing_vocab_and_last_commit(N):
    start = N.device_bytes()
    ctx = N.Context(device_id=0)                               # its own context: search workspaces are freed with it
    rng = np.random.default_rng(1)
    h = History(ctx, "adds")
    try:
        h.add(rows(rng, 3000, 1500))
        h.ix.commit(1500)
        assert N.last_commit()["merged"] == 0                 # no base yet: a full build
        for _ in range(4):                                    # single-row adds, one commit each
            h.add(rows(rng, 1, 1500))
            h.ix.commit(1500)
            lc = N.last_commit()
            assert lc["merged"] == 1 and lc["postings_written"] == h.ix.stats().nnz and lc["delta_entries"] >= 1
        h.add(rows(rng, 40, 1500, empty_every=2))             # rows with empty term lists
        h.ix.commit(1500)
        checkpoint(h, 1500)
        x, off, tid, tf, dl = rows(rng, 300, 1000)
        h.add((x, off, tid + 1500, tf, dl))                   # new term ids: vocab grows
        h.ix.commit(2600)
        assert N.last_commit()["merged"] == 1
        checkpoint(h, 2600)
        h.ix.commit(2600)                                     # nothing changed
        checkpoint(h, 2600)
    finally:
        h.ix.drop()
        ctx.close()
    assert N.device_bytes() == start


def test_removals(N, ctx):
    rng = np.random.default_rng(2)
    V = 2000
    h = History(ctx, "rm")
    try:
        ids = h.add(rows(rng, 5000, V))
        h.ix.commit(V)
        h.remove(rng.choice(ids, 400, replace=False))          # committed rows
        h.ix.commit(V)
        checkpoint(h, V)
        new = h.add(rows(rng, 700, V))
        h.remove(new[::3])                                     # rows added since the last commit
        h.remove(ids[:50])
        checkpoint(h, V)
        live = [i for op in h.log if op[0] == "add" for i in op[1]]
        h.remove(np.array(live, np.uint64))                    # every row
        h.ix.commit(V)
        assert h.ix.stats().nnz == 0 and h.ix.stats().n_docs_global == 0
        h.add(rows(rng, 900, V))                               # and adds again
        checkpoint(h, V)
    finally:
        h.ix.drop()


def test_rare_threshold_and_subtile_boundary(N, ctx):
    rng = np.random.default_rng(3)
    V, T = 3000, 2999                                          # term T: in chosen rows only
    h = History(ctx, "rare")

    def batch(n, with_t):
        x, off, tid, tf, dl = rows(rng, n, V - 1, extra=T if with_t else None)
        return x, off, tid, tf, dl
    try:
        h.add(batch(2000, True))
        h.add(batch(40, False))                                # 2040 rows: one sub-tile of 2048
        h.ix.commit(V)
        assert h.ix.read_postings(T)[2] == 2000
        with_t = h.add(batch(100, True))                       # df(T) 2100 > BM25_RARE_MAX, n_rows crosses 2048
        h.ix.commit(V)
        assert h.ix.read_postings(T)[2] == 2100 > RARE_MAX and h.ix.stats().n_rows > SUB_DOCS
        checkpoint(h, V)
        first = [op[1] for op in h.log if op[0] == "add"][0]
        h.remove(np.concatenate([first[:60], with_t[:10]]))   # back down to 2030
        h.ix.commit(V)
        assert h.ix.read_postings(T)[2] == 2030 <= RARE_MAX
        checkpoint(h, V)
    finally:
        h.ix.drop()


def test_long_term_over_several_delta_ranges(N, ctx, monkeypatch):
    """a term with > 1M postings, removals inside it, and a delta sorted in several term ranges"""
    monkeypatch.setenv("KRAG_BM25_BUILD_CHUNK", str(1 << 15))
    rng = np.random.default_rng(4)
    V, n = 500, 1_050_000
    h = History(ctx, "long")
    try:
        x = rng.standard_normal((n, DIM), dtype=np.float32)
        lens = rng.integers(0, 3, n)                           # term 0 and up to two other distinct terms per row
        a = rng.integers(1, V, n)
        b = rng.integers(1, V - 1, n)
        b = np.where(b >= a, b + 1, b)
        off = np.concatenate([[0], np.cumsum(1 + lens)]).astype(np.int64)
        tid = np.zeros(off[-1], np.uint32)
        tid[off[:-1][lens >= 1] + 1] = a[lens >= 1]
        tid[off[:-1][lens == 2] + 2] = b[lens == 2]
        tf = rng.integers(1, 4, tid.size).astype(np.uint16)
        dl = np.diff(off).astype(np.uint32) + 3
        ids = h.add((x, off, tid, tf, dl))
        h.ix.commit(V)
        assert h.ix.read_postings(0, cap=n + 1)[2] == n
        h.remove(rng.choice(ids, n // 100, replace=False))
        h.add(rows(rng, 60_000, V, extra=0))
        h.ix.commit(V)
        assert N.last_commit()["merged"] == 1
        checkpoint(h, V, terms=range(V))
    finally:
        h.ix.drop()


def _shard_commit(pair, vocab, inflate=(0, 0), local=True, cached=None):
    if local or cached is None:
        res = [ix.commit_local(vocab) for ix in pair]
    else:
        res = cached
    df = np.sum([r[0] for r in res], axis=0).astype(np.uint32)
    n_docs = sum(r[1] for r in res) + inflate[0]
    total = sum(r[2] for r in res) + inflate[1]
    for s, ix in enumerate(pair):
        ix.commit_global(vocab, df, n_docs, total, s)
    return res


def test_two_round_robin_shards(N, ctx):
    """shards 0 and 1 of a stride-2 ordinal map on one device: commit_local / commit_global with summed statistics"""
    rng = np.random.default_rng(5)
    V = 1500
    hs = [History(ctx, f"s{s}") for s in range(2)]
    for s, h in enumerate(hs):
        h.ix.set_ordinal_map(s, 2)

    def add(n):
        x, off, tid, tf, dl = rows(rng, n, V)
        for s, h in enumerate(hs):
            sel = np.arange(s, n, 2)
            lo, hi = off[sel], off[sel + 1]
            o = np.concatenate([[0], np.cumsum(hi - lo)]).astype(np.int64)
            take = np.concatenate([np.arange(a, b) for a, b in zip(lo, hi)]).astype(np.int64) if o[-1] else np.zeros(0, np.int64)
            h.add((x[sel], o, tid[take], tf[take], dl[sel]), ids=np.arange(h.next_id, h.next_id + sel.size, dtype=np.uint64) * 2 + s)
            h.next_id += sel.size

    def compare(inflate=(0, 0)):
        twins = []
        for s, h in enumerate(hs):
            t = h.ctx.create_index(f"t{s}", DIM)
            t.set_ordinal_map(s, 2)
            for op in h.log:
                t.add(op[1], *op[2]) if op[0] == "add" else t.remove(op[1])
            twins.append(t)
        try:
            _shard_commit(twins, V, inflate)
            for h, t in zip(hs, twins):
                assert_same_index(h.ix, t, V)
        finally:
            for t in twins:
                t.drop()

    try:
        add(4000)
        _shard_commit([h.ix for h in hs], V)
        add(301)
        for h in hs:
            h.remove(np.array([op[1] for op in h.log if op[0] == "add"][0][:40:3]))
        _shard_commit([h.ix for h in hs], V)
        assert N.last_commit()["merged"] == 1
        compare()
        add(77)
        _shard_commit([h.ix for h in hs], V, inflate=(5000, 123457))   # externally inflated global statistics
        compare(inflate=(5000, 123457))
        add(50)
        res = [h.ix.commit_local(V) for h in hs]
        hs[1].ix.commit_local(V + 1)           # shard 1's preparation is now for another vocab: its commit_global recomputes it
        _shard_commit([h.ix for h in hs], V, local=False, cached=res)
        compare()
    finally:
        for h in hs:
            h.ix.drop()


def test_rejected_commit_then_valid(N, ctx):
    rng = np.random.default_rng(6)
    h = History(ctx, "rej")
    try:
        h.add(rows(rng, 2000, 1000))
        h.ix.commit(1000)
        x, off, tid, tf, dl = rows(rng, 50, 100)
        h.add((x, off, tid + 1000, tf, dl))
        with pytest.raises(N.KragError) as e:
            h.ix.commit(1000)                                  # vocab <= largest term id
        assert e.value.code == N.KRAG_E_INVALID and not h.ix.stats().committed
        checkpoint(h, 1100)
        assert N.last_commit()["merged"] == 0                  # the twin's commit was the last one
    finally:
        h.ix.drop()


def test_persist_load_add_commit(N, ctx, tmp_path):
    rng = np.random.default_rng(7)
    V = 1200
    h = History(ctx, "pl")
    try:
        ids = h.add(rows(rng, 3000, V))
        h.ix.commit(V)
        h.remove(ids[::7])
        h.ix.commit(V)
        h.ix.persist(str(tmp_path))
        L = ctx.load_index("pl_loaded", str(tmp_path))
        assert N.last_commit()["merged"] == 0                  # load: one full build
        h.ix.drop()
        h.ix = L
        h.add(rows(rng, 500, V))
        h.ix.commit(V)
        assert N.last_commit()["merged"] == 1
        checkpoint(h, V, device_bytes=False)                   # the loaded index's buffers have their exact sizes
    finally:
        h.ix.drop()


def _live_rebuild_log(h):
    """the log of a fresh index holding h's live rows in order (what compaction leaves)"""
    removed = set()
    for op in h.log:
        if op[0] == "remove":
            removed.update(int(i) for i in op[1])
    out = []
    for op in h.log:
        if op[0] != "add":
            continue
        ids, (x, off, tid, tf, dl) = op[1], op[2]
        sel = np.array([i for i in range(ids.size) if int(ids[i]) not in removed], np.int64)
        if sel.size == 0:
            continue
        take = np.concatenate([np.arange(off[i], off[i + 1]) for i in sel]).astype(np.int64)
        o = np.concatenate([[0], np.cumsum(np.diff(off)[sel])]).astype(np.int64)
        out.append(("add", ids[sel], (x[sel], o, tid[take], tf[take], dl[sel])))
    return out


@pytest.mark.parametrize("committed", [True, False])
def test_compaction_then_adds(N, ctx, committed):
    rng = np.random.default_rng(8)
    V = 1500
    h = History(ctx, "cmp")
    try:
        ids = h.add(rows(rng, 6000, V))
        h.ix.commit(V)
        h.remove(rng.choice(ids, 1500, replace=False))
        if committed:
            h.ix.commit(V)
        else:
            new = h.add(rows(rng, 400, V))                     # added since the base, some of them removed
            h.remove(new[::4])
        assert h.ix.compact() > 0
        assert N.last_compact()["postings_ms"] > 0
        assert h.ix.stats().committed == committed
        h.log = _live_rebuild_log(h)
        if committed:
            checkpoint(h, V, device_bytes=False)               # the remapped postings alone
        h.add(rows(rng, 300, V))
        h.remove(h.log[0][1][:20])
        h.ix.commit(V)
        assert N.last_commit()["merged"] == 1
        checkpoint(h, V, device_bytes=False)
    finally:
        h.ix.drop()


def test_large_synthetic_index(N):
    """3M synthetic rows (vocab 2^20) plus 10k adds and 1 % removes: 2,000 sampled terms with the 50 most frequent, and a
    256-query retrieve"""
    start = N.device_bytes()
    V, n = 1 << 20, 3_000_000
    rng = np.random.default_rng(9)
    ctx = N.Context(device_id=0)
    A = ctx.create_index("big", DIM)
    T = None
    try:
        A.synth_fill(n, 0, 11, V)
        A.commit(V)
        x, off, tid, tf, dl = rows(rng, 10_000, V, mean_len=30)
        add_ids = np.arange(n, n + 10_000, dtype=np.uint64)
        dead = rng.choice(n + 10_000, (n + 10_000) // 100, replace=False).astype(np.uint64)
        A.add(add_ids, x, off, tid, tf, dl)
        A.remove(dead)
        A.commit(V)
        assert N.last_commit()["merged"] == 1
        T = ctx.create_index("big_twin", DIM)
        T.synth_fill(n, 0, 11, V)
        T.add(add_ids, x, off, tid, tf, dl)
        T.remove(dead)
        df = T.commit_local(V)[0]
        T.commit(V)
        assert N.last_commit()["merged"] == 0
        top = np.argsort(df, kind="stable")[-50:]
        terms = np.unique(np.concatenate([top, rng.integers(0, V, 1950), np.unique(tid)[:100]]))
        assert_same_index(A, T, V, terms=terms, seed=10)
        q = rng.standard_normal((256, DIM), dtype=np.float32)
        qt = [np.unique((rng.zipf(1.3, int(rng.integers(2, 8))) - 1) % V).astype(np.uint32) for _ in range(256)]
        ra, rb = A.retrieve(q, qt, 10), T.retrieve(q, qt, 10)
        for k in ra:
            assert same_arrays(ra[k], rb[k]), k
    finally:
        A.drop()
        if T is not None:
            T.drop()
        ctx.close()
    assert N.device_bytes() == start
