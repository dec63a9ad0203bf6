"""K3 (BM25) at the shard size where the default kernel choice takes bm25_warp_kernel, bit-exact against the CPU oracle.

Shards of 3,000,000 rows or more (BW_AUTO_MIN_ROWS in bm25.cu) run the warp kernel by default: a sample pass over every
`stride`-th 2048-document sub-tile, a threshold select, a main pass over all sub-tiles and a final select, with the
first-generation tile kernel as the exact safety net for queries whose candidate list overflowed.  Every other K3 test
forces the warp kernel on corpora of at most 400k documents, where the sample pass visits a handful of sub-tiles and can
never overflow its candidate list.  Here one index of N = 3,001,234 documents runs under the default choice:

- 1,466 sub-tiles, the last one partial (914 documents), and they do not fill the last 8-sub-tile work unit;
- dense rows of d = 64 (768 MB, split rows) so that the hybrid retrieve runs too;
- the term lists of oracle.synth_sparse (vocabulary 2^17, mean length 12) plus crafted terms, each aimed at one branch:
  T_ALL (every document: the sample list overflows), T_BURST (sub-tiles with more rounds than a staging buffer holds,
  between ordinary ones), T_TIE and T_TIE8 (200,000 and 25,000 equal scores starting at a sampled sub-tile, in every
  document and in every 8th: claimed by the sweep and out of the staging buffer), T_EDGE_RARE / T_EDGE_TILE
  (df 2048 and 2049: a per-batch resolve row and a tile-index row) and T_LAST (only in the partial last sub-tile).

Every search runs three times, under the default choice, KRAG_BM25_KERNEL=warp and KRAG_BM25_KERNEL=legacy.  The kernel
launch count of the default run must equal the warp run's and differ from the legacy run's, which proves that the
default took the warp kernel; all three results must equal the oracle bit for bit.  The oracle's top-P is a prefix of
its top-1024 (one total order: score desc, ordinal asc), so each query is computed once at 1024 and sliced.

The index is module-scoped.  The tombstone test removes rows for good, so it is the last test of the file.  On one H100
80GB HBM3 (700 W power limit) with 8 host cores the file runs in about 63 s, most of it in the CPU oracle (the dense top-P
of two 256-query batches over 3M rows); the index holds 1.4 GiB of device memory, the process 2.3 GiB with the search
workspaces."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
if not pytest.importorskip("torch").cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

N, D, SEED = 3_001_234, 64, 71
VOCAB0 = 2 ** 17                                   # synth_sparse's vocabulary; the crafted terms follow it
T_ALL, T_BURST, T_TIE, T_TIE8, T_EDGE_RARE, T_EDGE_TILE, T_LAST = range(VOCAB0, VOCAB0 + 7)
VOCAB = VOCAB0 + 7
SUB = 2048                                         # BM25_SUB_DOCS: one warp's accumulator range
N_SUB = (N + SUB - 1) // SUB                       # 1466
RARE_MAX = 2048                                    # BM25_RARE_MAX: longer lists have a tile-index row
STAGE_ROUNDS = 12                                  # BW_STAGE_ROUNDS: 32-posting rounds per staging buffer
BURST_SUBS = (5, 6, 13)                            # work units 0 and 1 (8 sub-tiles each) mix long and ordinary sub-tiles
TIE_LO, TIE_N, TIE_DL = 2 * 64 * SUB, 200_000, 16  # starts at sub-tile 128, sampled at stride 64
LAST_LO = (N // SUB) * SUB                         # first row of the partial last sub-tile
PMAX = 1024                                        # KRAG_MAX_POOL
AUTO_MIN_ROWS = 3_000_000                          # BW_AUTO_MIN_ROWS

assert N >= AUTO_MIN_ROWS and N % SUB and N_SUB % 8 and N_SUB == 1466


def _capq(P):
    """bm25.cu bw_capq without KRAG_BM25_CAPQ"""
    c = 32768
    while c < 256 * P and c < 262144:
        c <<= 1
    return c


def _stride(P, capq):
    """sample stride of the warp kernel's first pass (launch_bm25)"""
    return max(1, min(64, capq // (4 * P), N_SUB))


def _corpus(o):
    """(x, csr, postings) of the fixture: synth_sparse's lists with the crafted terms appended to chosen documents"""
    x = o.synth_dense(N, D, SEED)
    off, ids, tf, dl = o.synth_sparse(N, VOCAB0, SEED + 1, mean_len=12)
    dl = dl.copy()
    dl[TIE_LO:TIE_LO + TIE_N] = TIE_DL                    # equal length and tf 1: equal T_TIE scores
    rng = np.random.default_rng(SEED + 2)
    ex = []

    def put(rows, term, tfs=1):
        rows = np.asarray(rows, np.int64)
        ex.append((rows, np.full(rows.size, term, np.uint32), np.broadcast_to(np.asarray(tfs, np.uint16), rows.shape)))

    put(np.arange(N), T_ALL)
    burst = np.concatenate([np.arange(s * SUB, (s + 1) * SUB) for s in BURST_SUBS])
    # tf grows along a burst sub-tile, so the best documents sit in its last staged blocks
    put(burst, T_BURST, 1 + (burst % SUB) // 256)
    put(np.setdiff1d(np.nonzero(rng.random(N) < 0.01)[0], burst), T_BURST)
    put(np.arange(TIE_LO, TIE_LO + TIE_N), T_TIE)
    put(np.arange(TIE_LO, TIE_LO + TIE_N, 8), T_TIE8)                  # 256 postings = 8 rounds per sub-tile
    for term, df in ((T_EDGE_RARE, RARE_MAX), (T_EDGE_TILE, RARE_MAX + 1)):
        rows = np.unique(np.linspace(0, N - 1, df).astype(np.int64))     # first and last row included
        assert rows.size == df
        put(rows, term, 1 + np.arange(df) % 3)
    last = np.arange(LAST_LO, N, 2)
    put(last, T_LAST, 1 + np.arange(last.size) % 4)

    ed = np.concatenate([e[0] for e in ex])
    et = np.concatenate([e[1] for e in ex])
    ef = np.concatenate([e[2] for e in ex])
    order = np.lexsort((et, ed))
    ed, et, ef = ed[order], et[order], ef[order]
    cnt = np.bincount(ed, minlength=N)
    base_len = np.diff(off)
    off2 = np.zeros(N + 1, np.int64)
    off2[1:] = np.cumsum(base_len + cnt)
    ids2 = np.empty(off2[-1], np.uint32)
    tf2 = np.empty(off2[-1], np.uint16)
    pos = np.arange(ids.size, dtype=np.int64) + np.repeat(off2[:-1] - off[:-1], base_len)
    ids2[pos], tf2[pos] = ids, tf
    ex_first = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    pos = off2[ed] + base_len[ed] + (np.arange(ed.size) - ex_first[ed])
    ids2[pos], tf2[pos] = et, ef
    csr = (off2, ids2, tf2, dl)
    return x, csr, o.bm25_build(*csr, VOCAB)


class Fixture:
    def __init__(self, ctx, o):
        from kaito_b200 import _native
        self.ctx, self.o = ctx, o
        self.x, self.csr, self.post = _corpus(o)
        before = _native.device_bytes()
        self.ix = ctx.create_index("bm25_warp_scale", D)
        self.ix.add(np.arange(N, dtype=np.uint64), self.x, *self.csr)
        self.ix.commit(VOCAB)
        self.index_bytes = _native.device_bytes() - before
        self.df = np.diff(self.post.off)
        self._memo = {}

    def ref(self, qs, alive=None, tag=None):
        """oracle top-PMAX (score, ordinal) of each query, memoised per (tombstone set, query)"""
        keys = [(tag, tuple(int(t) for t in q)) for q in qs]
        todo = [(k, q) for k, q in zip(keys, qs) if k not in self._memo]

        def one(q):
            q = np.asarray(q, np.uint32)
            return self.o.bm25_query(self.post, q[q < VOCAB], PMAX, alive)

        with ThreadPoolExecutor(os.cpu_count() or 1) as pool:        # the oracle call releases the GIL
            for (k, _), r in zip(todo, pool.map(one, [q for _, q in todo])):
                self._memo[k] = r
        score = np.stack([self._memo[k][0] for k in keys])
        ordn = np.stack([self._memo[k][1] for k in keys])
        return score, ordn


@pytest.fixture(scope="module")
def fx(ctx, oracle):
    from kaito_b200 import _native
    f = Fixture(ctx, oracle)
    yield f
    print(f"device memory: index {f.index_bytes / 2**30:.2f} GiB, process {_native.device_bytes() / 2**30:.2f} GiB")
    f.ix.drop()


def _bench_batch(o):
    """256 queries as the bench draws them (rank_offset 0 and 20), with duplicated terms, out-of-vocabulary ids, and
    queries of 32, 33, 40 and 70 terms (more than 32 terms: the accumulate-all-then-sweep path)"""
    qs = o.synth_query_terms(VOCAB0, 128, seed=SEED + 3, rank_offset=0)
    qs += o.synth_query_terms(VOCAB0, 128, seed=SEED + 4, rank_offset=20)
    g = np.random.default_rng(SEED + 5)
    qs[0] = np.concatenate([qs[0], qs[0][:2], qs[0][:1]])
    qs[1] = np.array([VOCAB + 5, qs[1][0], 2 ** 32 - 1], np.uint32)
    for i, m in zip((2, 3, 4, 5), (32, 33, 40, 70)):
        qs[i] = g.integers(0, 3000, m).astype(np.uint32)
    qs[6] = np.concatenate([qs[6], qs[6][::-1]])
    return qs


def _with_filler(fx, special):
    """the special queries followed by bench queries up to the bench batch of 256"""
    return list(special) + _bench_batch(fx.o)[len(special):]


def _on_each_kernel(monkeypatch, ctx, call, default="warp"):
    """call() under the default kernel choice, KRAG_BM25_KERNEL=warp and =legacy.  The default run's launch count must
    equal that of the kernel the default is expected to take, and differ from the other's (the warp kernel's passes and
    selects launch more kernels than the first-generation kernel alone)."""
    res, launches = {}, {}
    for kern in ("auto", "warp", "legacy"):
        with monkeypatch.context() as m:
            if kern == "auto":
                m.delenv("KRAG_BM25_KERNEL", raising=False)
            else:
                m.setenv("KRAG_BM25_KERNEL", kern)
            c0 = ctx.launch_count()
            res[kern] = call()
            launches[kern] = ctx.launch_count() - c0
    other = "legacy" if default == "warp" else "warp"
    assert launches["auto"] == launches[default] and launches["warp"] > launches["legacy"], launches
    assert launches["auto"] != launches[other], launches
    return res


def _bm25_vs_oracle(fx, monkeypatch, qs, pools, alive=None, tag=None, ord_of=lambda r: r):
    rs, ro = fx.ref(qs, alive, tag)
    for P in pools:
        res = _on_each_kernel(monkeypatch, fx.ctx, lambda: fx.ix.search_bm25(qs, P))
        want_o = np.where(ro[:, :P] >= 0, ord_of(ro[:, :P]), -1)
        for kern, (score, ordn) in res.items():
            bad = np.nonzero((ordn != want_o).any(1) | (score.view(np.uint32) != rs[:, :P].view(np.uint32)).any(1))[0]
            assert bad.size == 0, f"{kern} P={P}: queries {bad[:8].tolist()} differ from the oracle"
    return rs, ro


# ------------------------------------------------------------------------------------------------------------- cases
def test_postings_and_kernel_choice(fx, ctx, oracle, monkeypatch):
    """postings of the crafted terms bit-exact; the 3M-row boundary: the default choice takes the warp kernel on the
    fixture and the first-generation kernel on a shard of AUTO_MIN_ROWS - 1 rows"""
    assert fx.index_bytes < 4 << 30, fx.index_bytes
    assert fx.df[T_ALL] == N and fx.df[T_TIE] == TIE_N and fx.df[T_LAST] == (N - LAST_LO + 1) // 2
    assert fx.df[T_EDGE_RARE] == RARE_MAX and fx.df[T_EDGE_TILE] == RARE_MAX + 1
    for t in (T_ALL, T_BURST, T_TIE, T_TIE8, T_EDGE_RARE, T_EDGE_TILE, T_LAST, 0, 1, 2, 3, VOCAB0 - 1):
        docs, scores, cnt = fx.ix.read_postings(t)
        sl = slice(fx.post.off[t], fx.post.off[t + 1])
        assert cnt == fx.df[t], t
        assert np.array_equal(docs, fx.post.doc[sl]) and np.array_equal(scores, fx.post.score[sl]), t
    assert (fx.post.doc[fx.post.off[T_LAST]:fx.post.off[T_LAST + 1]] >= LAST_LO).all()

    qs = [np.array([T_EDGE_RARE, 7], np.uint32), np.array([T_EDGE_TILE], np.uint32)] * 2
    _bm25_vs_oracle(fx, monkeypatch, qs, (30,))

    # companion shard one row below the boundary: the first AUTO_MIN_ROWS - 1 documents with one short term each
    n2 = AUTO_MIN_ROWS - 1
    small = ctx.create_index("bm25_below_auto_min", 32)
    try:
        off = np.arange(n2 + 1, dtype=np.int64)
        tids = (np.arange(n2) % 1000).astype(np.uint32)
        small.add(np.arange(n2, dtype=np.uint64), np.ascontiguousarray(fx.x[:n2, :32]), off, tids,
                  np.ones(n2, np.uint16), fx.csr[3][:n2])
        small.commit(1000)
        qs2 = [np.array([3, 999], np.uint32), np.array([5], np.uint32)]
        post2 = oracle.bm25_build(off, tids, np.ones(n2, np.uint16), fx.csr[3][:n2], 1000)
        res = _on_each_kernel(monkeypatch, ctx, lambda: small.search_bm25(qs2, 30), default="legacy")
        for kern, (score, ordn) in res.items():
            for b, qt in enumerate(qs2):
                rs, ro = oracle.bm25_query(post2, qt, 30)
                assert np.array_equal(ordn[b], ro) and np.array_equal(score[b], rs), (kern, b)
    finally:
        small.drop()


@pytest.mark.parametrize("P", [1, 30, 90, 900, 1024])
def test_bench_batch(fx, monkeypatch, P):
    """The bench's batch shape (256 queries, about 47k work units per pass) at the service's pool sizes"""
    _bm25_vs_oracle(fx, monkeypatch, _bench_batch(fx.o), (P,))


@pytest.mark.parametrize("P", [128, 129, 256, 257, 512, 513])
def test_pool_sizes_that_change_capq_and_stride(fx, monkeypatch, P):
    """The candidate-list capacity doubles past P = 128, 256 and 512 (bw_capq), and with it the sample select's
    input and the share of the list the main pass may fill.  The sample stride capq // (4 P) stays at its cap of 64
    (capq >= 256 P); test_safety_net_at_scale runs stride 1."""
    assert P % 2 == 0 or _capq(P) == 2 * _capq(P - 1)
    assert _stride(P, _capq(P)) == 64
    _bm25_vs_oracle(fx, monkeypatch, _bench_batch(fx.o), (P,))


def test_sample_list_overflow(fx, monkeypatch):
    """Queries whose sample pass pushes more keys than the candidate list holds.  At P = 30 the list holds
    capq = 32,768 keys and the sample stride is min(64, 32768 // 120) = 64, so the sample pass visits sub-tiles
    0, 64, ..., 1408: ceil(1466 / 64) = 23 sub-tiles, all full (1409 * 2048 <= N).  T_ALL is in every document, so a
    query containing it pushes 23 * 2048 = 47,104 keys: cand_cnt exceeds capq after the sample pass, and mode 0 of
    bm25_select_kernel takes its threshold from whichever 32,768 keys landed first.  The same count is computed below
    from the oracle's postings for every query of the case, the four most frequent terms included."""
    P = 30
    capq = _capq(P)
    stride = _stride(P, capq)
    assert (capq, stride) == (32768, 64)
    rare = np.nonzero((fx.df[:VOCAB0] > 0) & (fx.df[:VOCAB0] <= 40))[0][:6].astype(np.uint32)
    special = [np.array([T_ALL], np.uint32),
               np.concatenate([[T_ALL], rare[:3]]).astype(np.uint32),
               np.concatenate([rare[3:], [T_ALL]]).astype(np.uint32),
               np.array([0, 1, 2, 3], np.uint32),
               np.array([3, T_ALL, 2], np.uint32)]
    sampled = np.zeros(N, bool)
    for s in range(0, N_SUB, stride):
        sampled[s * SUB:(s + 1) * SUB] = True
    for q in special:
        touched = np.zeros(N, bool)
        for t in q:
            touched[fx.post.doc[fx.post.off[t]:fx.post.off[t + 1]]] = True
        assert (touched & sampled).sum() > capq, q
    _bm25_vs_oracle(fx, monkeypatch, _with_filler(fx, special), (P,))


@pytest.mark.parametrize("P", [30, 900])
def test_long_sub_tiles(fx, monkeypatch, P):
    """T_BURST gives sub-tiles 5, 6 and 13 64 rounds of postings (more than a staging buffer's 12), between
    sub-tiles of one round, inside work units 0 and 1.  Those sub-tiles are accumulated block by block and claimed by
    bw_claim_sweep; the next sub-tile's prefetch (cp_async_wait<1>) and the buffer toggle cross both branches.  tf
    grows along a burst sub-tile, so the best documents are in its last staged blocks."""
    rounds = [-(-int(np.count_nonzero(fx.post.doc[fx.post.off[T_BURST]:fx.post.off[T_BURST + 1]] // SUB == s)) // 32)
              for s in range(16)]
    assert all(rounds[s] > STAGE_ROUNDS for s in BURST_SUBS)
    assert all(0 < rounds[s] <= STAGE_ROUNDS for s in range(16) if s not in BURST_SUBS), rounds
    special = [np.array([T_BURST], np.uint32),
               np.array([T_BURST, 5, 100, 2000], np.uint32),
               np.array([17, T_BURST, 300], np.uint32),
               np.array([T_BURST, T_EDGE_RARE, T_BURST], np.uint32)]
    rs, ro = _bm25_vs_oracle(fx, monkeypatch, _with_filler(fx, special), (P,))
    top = ro[0, :30]                                  # T_BURST alone: its best documents lie past the first staged block
    assert (top // SUB == BURST_SUBS[0]).all() and (top % SUB >= STAGE_ROUNDS * 32).all(), top


@pytest.mark.parametrize("P", [1, 30, 1024])
def test_ties_at_the_threshold(fx, monkeypatch, P):
    """T_TIE scores 200,000 documents equally, T_TIE8 every 8th of them, in sampled and unsampled sub-tiles
    alike.  T_TIE's sub-tiles have 64 rounds (claimed by bw_claim_sweep), T_TIE8's 8 (claimed out of the staging buffer).
    The sampled threshold is the key of the block's P-th document: the main pass must admit exactly the keys <= it, i.e.
    the block's lowest P ordinals (with fewer than P sampled documents, at P = 1024 for T_TIE8, there is no threshold)."""
    qs = _with_filler(fx, [np.array([T_TIE], np.uint32), np.array([T_TIE8], np.uint32), np.array([T_TIE], np.uint32)])
    rs, ro = _bm25_vs_oracle(fx, monkeypatch, qs, (P,))
    for b, step in ((0, 1), (1, 8)):
        assert np.array_equal(ro[b, :P], TIE_LO + step * np.arange(P)) and (rs[b, :P] == rs[b, 0]).all(), b


def test_safety_net_at_scale(fx, monkeypatch):
    """KRAG_BM25_CAPQ=64 on a 256-query batch.  The sample stride is then 1 (64 // 120 = 0), so the sample pass
    pushes every document a query touches.  The broad queries touch about 10^5 or more documents: their lists overflow,
    the threshold is the 30th best of 64 of their documents, and the main pass overflows again; bm25_tile_kernel then
    recomputes only those (its `only` flags) over 23 groups of 8 16,384-document tiles and launch_merge merges them.  The
    narrow queries touch at most 64 documents and stay on the warp kernel."""
    monkeypatch.setenv("KRAG_BM25_CAPQ", "64")
    assert -(-N // (SUB * 8)) == 184 and 184 // 8 == 23
    seen = np.nonzero(fx.df[:VOCAB0])[0]
    small = seen[np.argsort(fx.df[seen], kind="stable")[:24]].astype(np.uint32)   # the rarest terms: a few documents each
    narrow = [small[i:i + 2] for i in range(0, 24, 2)]
    assert all(0 < int(fx.df[q].sum()) <= 64 for q in narrow)
    qs = _bench_batch(fx.o)
    for i, q in enumerate(narrow):
        qs[20 * i + 7] = q
    broad = [q for i, q in enumerate(qs) if i % 20 != 7 and int(fx.df[q[q < VOCAB]].max(initial=0)) > 100_000]
    assert len(broad) > 100
    _bm25_vs_oracle(fx, monkeypatch, qs, (30,))


def test_ordinal_map(fx, monkeypatch):
    """set_ordinal_map(base=1, stride=3), as a round-robin shard: ordinals, and the order of ties, follow 1 + 3 r"""
    qs = _with_filler(fx, [np.array([T_TIE], np.uint32), np.array([T_LAST], np.uint32), np.array([T_ALL], np.uint32)])
    fx.ix.set_ordinal_map(1, 3)
    try:
        _bm25_vs_oracle(fx, monkeypatch, qs, (30, 1024), ord_of=lambda r: 1 + 3 * r)
    finally:
        fx.ix.set_ordinal_map(0, 1)


def _retrieve_vs_oracle(fx, monkeypatch, q, qs, k, alive=None, tag=None, **kw):
    o = fx.o
    P = o.pool_size(k)
    res = _on_each_kernel(monkeypatch, fx.ctx, lambda: fx.ix.retrieve(q, qs, k, **kw))
    dd, do = o.dense_topk(fx.x, q, P, alive)
    bs, bo = fx.ref(qs, alive, tag)
    for b in range(len(qs)):
        fin, de, sp, rk, od = o.fuse(dd[b], do[b], bs[b, :P], bo[b, :P], k)
        for kern, got in res.items():
            c = int(got["count"][b])
            assert c == len(od) and np.array_equal(got["ordinal"][b, :c], od), (kern, b)
            assert np.array_equal(got["final"][b, :c], fin), (kern, b)
            assert np.array_equal(got["rank"][b, :c], rk), (kern, b)
            assert np.array_equal(got["dense"][b, :c], de, equal_nan=True), (kern, b)
            assert np.array_equal(got["sparse"][b, :c], sp, equal_nan=True), (kern, b)


def test_hybrid_retrieve(fx, monkeypatch):
    """krag_retrieve at k = 10 on the bench batch: dense stage, K3 on the warp kernel, fuse"""
    q = fx.o.synth_queries(fx.x, 256, SEED + 6)
    _retrieve_vs_oracle(fx, monkeypatch, q, _bench_batch(fx.o), 10)


def test_tombstones_and_pushdown(fx, monkeypatch):
    """Last test of the file: the removals stay.  About 5 % of the rows die, among them the first rows of T_TIE's block and every
    document of the partial last sub-tile; then a hybrid retrieve with KRAG_FILTER_PUSHDOWN and an allow bitmap"""
    from kaito_b200 import _native
    o = fx.o
    rng = np.random.default_rng(SEED + 7)
    dead = np.unique(np.concatenate([np.nonzero(rng.random(N) < 0.05)[0], np.arange(TIE_LO, TIE_LO + 100),
                                     np.arange(LAST_LO, N)]))
    assert fx.ix.remove(dead.astype(np.uint64)) == dead.size
    alive = o.alive_bitmap(N, dead)
    assert np.array_equal(fx.ix.alive_bitmap()[:alive.size], alive)
    qs = _with_filler(fx, [np.array([T_TIE], np.uint32), np.array([T_LAST], np.uint32), np.array([T_ALL], np.uint32),
                           np.array([T_BURST, 9], np.uint32), np.array([T_LAST, T_EDGE_TILE], np.uint32)])
    rs, ro = _bm25_vs_oracle(fx, monkeypatch, qs, (30, 1024), alive, tag="dead")
    first_live = TIE_LO + 100 + np.nonzero(~np.isin(np.arange(TIE_LO + 100, TIE_LO + 200), dead))[0][:30]
    assert np.array_equal(ro[0, :30], first_live)
    assert (rs[1] == 0).all()                                     # T_LAST's documents are all dead: zero fill

    allow = np.packbits(rng.random(((N + 31) // 32) * 32) < 0.3, bitorder="little").view(np.uint32)
    q = o.synth_queries(fx.x, 256, SEED + 8)
    _retrieve_vs_oracle(fx, monkeypatch, q, _bench_batch(o), 10, alive=allow & alive, tag="pushdown",
                        fusion_mode=_native.FILTER_PUSHDOWN, keyword_allow_bitmap=allow)
