"""GPU edge cases of the dense kernels K1 (exact scan) and K2 (tensor-core prune + exact rescore + certificate) and of
K3 (BM25), bit-exact against the CPU oracle:

- an adversarial corpus on which the kernel's own bf16 rounding prunes the exact nearest row of one query, so only a
  sound certificate (and the K1 fallback it triggers) returns the right answer (construction: test_tc_certificate_bound.py);
- rows wider than 12 288 dimensions, whose exact rescoring needs more than 48 KB of shared memory;
- candidate pools at the select buffers' capacity boundaries and up to KRAG_MAX_POOL, batches around K1's query groups
  and K2's NQ buckets and 256-query chunks, odd dimensions;
- groups of bit-identical rows (and documents) spread over CTAs, epochs, tiles and query chunks: ties go to the lower
  ordinal, exactly as in the oracle.

Large corpora are module-scoped; every test that switches dense modes has its own Context."""
import numpy as np
import pytest

from tests import test_tc_certificate_bound as adv

pytestmark = pytest.mark.gpu

POOL_MAX = 1024


def _native():
    from kaito_b200 import _native
    return _native


def _fallbacks():
    return _native().load().krag_tc_fallback_queries()


def _assert_k2_ran(kid, fb, what):
    """the last dense kernel is the K2 prune pass, or K1 re-ran queries that K2 could not certify (the fallback counter
    only moves inside K2)"""
    got = _native().last_dense_kernel()[1]
    assert got == kid or (got == 1 and fb > 0), f"{what}: last dense kernel {got}, {fb} fallbacks"


def _assert_same(got, ref, what):
    (gd, go), (rd, ro) = got, ref
    assert np.array_equal(go, ro), f"{what}: ids differ (first bad query {np.nonzero((go != ro).any(1))[0][:5]})"
    assert np.array_equal(gd, rd), f"{what}: distances differ"


# ----------------------------------------------------------------------- (a) the certificate on adversarial rounding
@pytest.fixture(scope="module")
def adversarial():
    return {}


@pytest.mark.parametrize("P", [1, 10])
@pytest.mark.parametrize("mode", ["cvt", "bf16", "tf32"])
def test_tc_certificate_adversarial_rounding(oracle, adversarial, mode, P):
    """the adversarial query's exact nearest row is pruned by the bf16 main pass (TC_CVT, TC_BF16): the query must fail
    its certificate and be re-run on K1.  The TF32 pass admits the row.  Either way the answer equals the oracle."""
    N = _native()
    if P not in adversarial:
        x, q_adv, _ = adv.adversarial_corpus(P)
        q = np.concatenate([q_adv[None, :], oracle.synth_queries(x, 15, seed=40 + P)])
        adversarial[P] = (x, q, oracle.dense_topk(x, q, P))
    x, q, ref = adversarial[P]
    assert ref[1][0, 0] == adv.TARGET_ROW
    dense_mode, kid = {"cvt": (N.DENSE_TC, 5), "bf16": (N.DENSE_TC_BF16, 4), "tf32": (N.DENSE_TC_TF32, 3)}[mode]
    c = N.Context(device_id=0, dense_mode=dense_mode)
    try:
        ix = c.create_index(f"adv_{mode}_{P}", adv.D)
        ix.add(np.arange(adv.N, dtype=np.uint64), x)
        # the kernel's own sample-pass values (TF32) of the threshold rows lie inside the window the construction needs
        a = ix.debug_tc_dump(q[:1])[0]
        rows = adv.sampled_rows(adv.N)[::adv.TC_DUMP_GROUP]
        lo, hi = adv.threshold_window(x, q[0], P)
        assert lo < a[rows].min() and a[rows].max() < hi, (lo, a[rows].min(), a[rows].max(), hi)
        fb0 = _fallbacks()
        got = ix.search_dense(q, P)
        fb = _fallbacks() - fb0
        _assert_same(got, ref, f"K2 {mode} P={P}")
        _assert_k2_ran(kid, fb, f"K2 {mode} P={P}")
        if mode != "tf32":
            assert fb >= 1, "the pruned nearest row can only come back through the K1 fallback"
        ix.drop()
    finally:
        c.close()


# ------------------------------------------------------------------------------------------- (c) wide rows
@pytest.mark.parametrize("d", [12288, 12352, 16384])
def test_tc_wide_rows(oracle, d):
    """262 144 rows of 12 288 (the query row fills exactly 48 KB of shared memory in the rescoring kernel), 12 352 and
    16 384 dimensions, generated on the device: AUTO (K2, default pass) against the same index on K1"""
    N = _native()
    n, batch = adv.TC_MIN_ROWS, 32
    c = N.Context(device_id=0)
    try:
        ix = c.create_index(f"wide_{d}", d)
        ix.synth_fill(n, row_base=0, seed=d, vocab=0)
        picks = np.random.default_rng(d).integers(0, n, 48)
        xs = np.concatenate([ix.read_rows(int(r), 1) for r in picks])
        q = oracle.synth_queries(xs, batch, seed=d + 1)
        for P in (30, POOL_MAX):
            ix.set_dense_mode(N.DENSE_AUTO)
            fb0 = _fallbacks()
            got = ix.search_dense(q, P)
            _assert_k2_ran(5, _fallbacks() - fb0, f"d={d} P={P}")
            ix.set_dense_mode(N.DENSE_SCAN)
            ref = ix.search_dense(q, P)
            assert N.last_dense_kernel()[1] == 1
            _assert_same(got, ref, f"d={d} P={P}")
            for b in (0, batch - 1):          # planted and random query: distances re-derived on the CPU
                o = got[1][b, :30]
                rows = np.concatenate([ix.read_rows(int(r), 1) for r in o])
                assert np.array_equal(oracle.l2sq(rows, q[b]), got[0][b, :30])
            assert (np.diff(got[0], axis=1) >= 0).all()
        ix.drop()
    finally:
        c.close()


# ------------------------------------------------------------------------------- (d) pool, batch and dimension edges
K1_POOLS = (1, 2, 511, 512, 513, 1023, 1024)     # ds_cap switches from 1024 to 2048 entries above 512


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1_000_000])
def test_k1_pool_and_batch_edges(ctx_scan, oracle, n):
    """K1 with 1, 3 and 15 queries (query groups of 4/2/1 with remainders), pools around the select buffer's capacity;
    at 1M rows the epoch prune and the cross-CTA threshold hint fire several times"""
    d = 64
    x = oracle.synth_dense(n, d, seed=n + 3)
    q = oracle.synth_queries(x, 15, seed=n + 4)
    rd, ro = oracle.dense_topk(x, q, POOL_MAX)          # top-P is a prefix of top-1024 (total order: distance, ordinal)
    ix = ctx_scan.create_index(f"k1edge_{n}", d)
    try:
        ix.add(np.arange(n, dtype=np.uint64), x)
        for P in K1_POOLS:
            for batch in (1, 3, 15):
                got = ix.search_dense(q[:batch], P)
                assert _native().last_dense_kernel()[1] == 1
                _assert_same(got, (rd[:batch, :P], ro[:batch, :P]), f"K1 n={n} P={P} batch={batch}")
    finally:
        ix.drop()


@pytest.fixture(scope="module")
def corpus_300k(oracle):
    n, d = 300_000, 64
    x = oracle.synth_dense(n, d, seed=301)
    q = oracle.synth_queries(x, 257, seed=302)
    return x, q, oracle.dense_topk(x, q, POOL_MAX)


@pytest.mark.parametrize("mode", ["cvt", "tf32"])
def test_k2_pool_and_batch_edges(corpus_300k, mode):
    """K2 at P = 1 and KRAG_MAX_POOL for batches at and past its NQ buckets (64 / 128 / 256 queries per pass) and a
    257-query batch whose second 256-query chunk holds a single query"""
    N = _native()
    x, q, (rd, ro) = corpus_300k
    c = N.Context(device_id=0, dense_mode=N.DENSE_TC if mode == "cvt" else N.DENSE_TC_TF32)
    try:
        ix = c.create_index(f"k2edge_{mode}", x.shape[1])
        ix.add(np.arange(x.shape[0], dtype=np.uint64), x)
        for P in (1, POOL_MAX):
            for batch in (16, 64, 65, 128, 129, 256, 257):
                fb0 = _fallbacks()
                got = ix.search_dense(q[:batch], P)
                _assert_k2_ran(5 if mode == "cvt" else 3, _fallbacks() - fb0, f"K2 {mode} P={P} batch={batch}")
                _assert_same(got, (rd[:batch, :P], ro[:batch, :P]), f"K2 {mode} P={P} batch={batch}")
        ix.drop()
    finally:
        c.close()


def test_auto_switches_kernels_at_16_queries_with_identical_results(corpus_300k):
    """AUTO: 15 queries run on K1, 16 on K2; the 15 shared queries get identical rows and distances"""
    N = _native()
    x, q, (rd, ro) = corpus_300k
    c = N.Context(device_id=0)
    try:
        ix = c.create_index("auto_switch", x.shape[1])
        ix.add(np.arange(x.shape[0], dtype=np.uint64), x)
        for P in (30, POOL_MAX):
            d15, o15 = ix.search_dense(q[:15], P)
            assert N.last_dense_kernel()[1] == 1
            fb0 = _fallbacks()
            d16, o16 = ix.search_dense(q[:16], P)
            _assert_k2_ran(5, _fallbacks() - fb0, f"AUTO P={P}")
            assert np.array_equal(o15, o16[:15]) and np.array_equal(d15, d16[:15])
            _assert_same((d16, o16), (rd[:16, :P], ro[:16, :P]), f"AUTO P={P}")
        ix.drop()
    finally:
        c.close()


@pytest.mark.parametrize("d", [1, 31, 33, 96, 800])
def test_dense_odd_dimensions(oracle, d):
    """padded dimensions through K1 and K2; where dpad % 64 == 32 (d = 1, 31, 96, 800) the default mode runs the TF32
    prune pass (kernel 3), otherwise the bf16 pass (kernel 5).  d = 1: every unit row is +-1, so ties dominate."""
    N = _native()
    n, batch, P = adv.TC_MIN_ROWS, 16, 30
    x = oracle.synth_dense(n, d, seed=d + 7)
    q = oracle.synth_queries(x, batch, seed=d + 8)
    ref = oracle.dense_topk(x, q, P)
    dpad = (d + 31) // 32 * 32
    c = N.Context(device_id=0)
    try:
        ix = c.create_index(f"odd_{d}", d)
        ix.add(np.arange(n, dtype=np.uint64), x)
        fb0 = _fallbacks()
        got = ix.search_dense(q, P)
        _assert_k2_ran(5 if dpad % 64 == 0 else 3, _fallbacks() - fb0, f"d={d}")
        _assert_same(got, ref, f"K2 d={d}")
        ix.set_dense_mode(N.DENSE_SCAN)
        got = ix.search_dense(q, P)
        assert N.last_dense_kernel()[1] == 1
        _assert_same(got, ref, f"K1 d={d}")
        ix.drop()
    finally:
        c.close()


@pytest.fixture(params=["warp", "legacy"])
def bm25_kernel(request, monkeypatch):
    monkeypatch.setenv("KRAG_BM25_KERNEL", request.param)
    return request.param


def _sparse_index(ctx, oracle, name, n, vocab, d, seed, csr=None):
    x = oracle.synth_dense(n, d, seed)
    off, ids, tf, dl = csr if csr is not None else oracle.synth_sparse(n, vocab, seed + 1)
    ix = ctx.create_index(name, d)
    ix.add(np.arange(n, dtype=np.uint64), x, off, ids, tf, dl)
    ix.commit(vocab)
    return ix, x, oracle.bm25_build(off, ids, tf, dl, vocab)


def test_bm25_pool_edges_and_fused_pool(ctx_scan, oracle, bm25_kernel):
    """K3 at pools around its per-query buffer (256/257 and 512/513 entries) and KRAG_MAX_POOL, then a retrieve whose
    fused pool is 900 (k = 300, candidate multiplier 3)"""
    n, vocab, d = 40_000, 3000, 32
    ix, x, post = _sparse_index(ctx_scan, oracle, f"bm25edge_{bm25_kernel}", n, vocab, d, seed=51)
    try:
        qs = oracle.synth_query_terms(vocab, 6, seed=52, rank_offset=20)
        qs[0] = np.array([vocab - 1], np.uint32)                         # short list: zero-score fill up to P
        for P in (1, 256, 257, 512, 513, POOL_MAX):
            score, ordn = ix.search_bm25(qs, P)
            for b, qt in enumerate(qs):
                rs, ro = oracle.bm25_query(post, qt, P)
                assert np.array_equal(ordn[b], ro), (P, b)
                assert np.array_equal(score[b], rs), (P, b)
        k = 300
        P = oracle.pool_size(k)
        q = oracle.synth_queries(x, len(qs), seed=53)
        out = ix.retrieve(q, qs, k)
        for b in range(len(qs)):
            dd, do = oracle.dense_topk(x, q[b:b + 1], P)
            bs, bo = oracle.bm25_query(post, qs[b], P)
            fin, de, sp, rk, od = oracle.fuse(dd[0], do[0], bs, bo, k)
            cnt = int(out["count"][b])
            assert cnt == len(od) and np.array_equal(out["ordinal"][b, :cnt], od), b
            assert np.array_equal(out["final"][b, :cnt], fin) and np.array_equal(out["rank"][b, :cnt], rk)
    finally:
        ix.drop()


# ------------------------------------------------------------------------------------------------------ (e) ties
TIE_N, TIE_D = 300_000, 64


def _tie_groups(n, rng):
    """two groups of ordinals whose rows are made bit-identical.  Group A (1100 rows, more than any pool) spans every K1
    CTA (64-row tile t -> CTA t mod 264), both epochs of a 300 000-row K1 scan and many K2 tiles; group B (40 rows)
    straddles P = 30.  Fixed members: the first rows of CTAs 0, 1 and 263, CTA 0's second tile, the last rows."""
    fixed = np.array([3, 64 + 3, 263 * 64 + 3, 264 * 64 + 3, n - 1])
    a = np.unique(np.concatenate([fixed, rng.choice(n, 1100 - len(fixed), replace=False)]))
    rest = np.setdiff1d(np.arange(n), a)
    b = np.sort(rng.choice(rest, 40, replace=False))
    return a, b


@pytest.fixture(scope="module")
def tie_corpus(oracle):
    rng = np.random.default_rng(71)
    x = oracle.synth_dense(TIE_N, TIE_D, seed=72)
    ga, gb = _tie_groups(TIE_N, rng)
    x[ga] = x[ga[len(ga) // 2]]
    x[gb] = x[gb[-1]]
    near = lambda r: (x[r] + 1e-3 * rng.standard_normal(TIE_D).astype(np.float32)).astype(np.float32)
    q = oracle.synth_queries(x, 260, seed=73)
    # exact copies and nearby queries of both groups, at the start of the batch and on both sides of the 256-query chunk
    q[0], q[1], q[255], q[256], q[257], q[258] = x[ga[0]], near(ga[0]), x[gb[0]], near(gb[0]), x[ga[0]], near(ga[0])
    out = {"x": x, "q": q, "ga": ga, "gb": gb}
    for P in (30, POOL_MAX):
        out[P] = oracle.dense_topk(x, q, P)
    # the groups straddle position P, so ties decide which members come back: the lowest ordinals
    for j, g in ((0, ga), (1, ga), (255, gb), (256, gb)):
        assert np.array_equal(out[30][1][j], g[:30])
    assert np.array_equal(out[POOL_MAX][1][0], ga[:POOL_MAX])
    return out


@pytest.mark.parametrize("mode", ["scan", "cvt", "bf16", "tf32"])
def test_dense_ties_break_by_ordinal(tie_corpus, mode):
    N = _native()
    x, q = tie_corpus["x"], tie_corpus["q"]
    dense_mode = {"scan": N.DENSE_SCAN, "cvt": N.DENSE_TC, "bf16": N.DENSE_TC_BF16, "tf32": N.DENSE_TC_TF32}[mode]
    c = N.Context(device_id=0, dense_mode=dense_mode)
    try:
        ix = c.create_index(f"ties_{mode}", TIE_D)
        ix.add(np.arange(TIE_N, dtype=np.uint64), x)
        for P in (30, POOL_MAX):
            fb0 = _fallbacks()
            got = ix.search_dense(q, P)
            _assert_k2_ran({"scan": 1, "cvt": 5, "bf16": 4, "tf32": 3}[mode], _fallbacks() - fb0, f"ties {mode} P={P}")
            _assert_same(got, tie_corpus[P], f"ties {mode} P={P}")
            if mode != "scan":                       # the group's copy alone (K2 pads it to a 64-query pass; bf16: K1)
                one = ix.search_dense(q[:1], P)
                _assert_same(one, (tie_corpus[P][0][:1], tie_corpus[P][1][:1]), f"ties {mode} P={P} single")
        ix.drop()
    finally:
        c.close()


def test_bm25_ties_break_by_ordinal(ctx_scan, oracle, bm25_kernel):
    """1100 documents with identical terms (so bit-identical BM25 scores) spread over every K3 tile: a query of their
    terms returns the lowest ordinals first at P = 30 and 1024, as the oracle does"""
    n, vocab, d = 60_000, 4000, 32
    off, ids, tf, dl = oracle.synth_sparse(n, vocab, 81)
    rng = np.random.default_rng(82)
    grp = np.sort(rng.choice(n, 1100, replace=False))
    grp[0], grp[-1] = 0, n - 1
    grp = np.unique(grp)
    # the group's documents hold exactly: two terms no other document has, and one frequent term
    s_ids, s_tf = np.array([vocab - 1, vocab - 2, 5], np.uint32), np.array([2, 1, 3], np.uint16)
    doc_of = np.repeat(np.arange(n), np.diff(off))
    keep = ~np.isin(ids, s_ids[:2]) & ~np.isin(doc_of, grp)
    doc2 = np.concatenate([doc_of[keep], np.repeat(grp, 3)])
    order = np.argsort(doc2, kind="stable")
    ids2 = np.concatenate([ids[keep], np.tile(s_ids, len(grp))])[order]
    tf2 = np.concatenate([tf[keep], np.tile(s_tf, len(grp))])[order]
    off2 = np.concatenate([[0], np.cumsum(np.bincount(doc2, minlength=n))]).astype(np.int64)
    dl = dl.copy()
    dl[grp] = 40
    ix, x, post = _sparse_index(ctx_scan, oracle, f"bm25ties_{bm25_kernel}", n, vocab, d, seed=83,
                                csr=(off2, ids2, tf2, dl))
    try:
        qs = [np.array([vocab - 1], np.uint32), np.array([vocab - 2, 5], np.uint32), np.array([vocab - 1, vocab - 2, 7], np.uint32)]
        for P in (30, POOL_MAX):
            score, ordn = ix.search_bm25(qs, P)
            for b, qt in enumerate(qs):
                rs, ro = oracle.bm25_query(post, qt, P)
                assert np.array_equal(ordn[b], ro), (P, b)
                assert np.array_equal(score[b], rs), (P, b)
            assert np.array_equal(ordn[0], grp[:P])
    finally:
        ix.drop()
