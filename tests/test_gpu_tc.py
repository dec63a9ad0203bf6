"""GPU tests of K2, the wgmma prune kernel: raw tensor-core output against numpy, and the
full prune -> exact-rescore -> certify pipeline bit-exact against the oracle."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["cvt", "tf32"])
def ctx_tc(request):
    """K2 forced for every batch size: the default prune pass ("cvt": bf16 wgmma on the high halves of split rows, TF32
    on rows with dpad % 64 == 32) and the TF32 pass (tf32 wgmma)"""
    from kaito_b200 import _native
    c = _native.Context(device_id=0, dense_mode=_native.DENSE_TC if request.param == "cvt" else _native.DENSE_TC_TF32)
    yield c
    c.close()


@pytest.mark.parametrize("n,d,nq", [(128, 32, 3), (1000, 64, 5), (777, 768, 100), (4096, 384, 256), (130, 1024, 64)])
def test_tc_raw_output_matches_numpy(ctx_tc, oracle, request, n, d, nq):
    from kaito_b200 import _native
    from tests import test_gpu_tc_passes as passes
    x = oracle.synth_dense(n, d, seed=n + d)
    q = oracle.synth_queries(x, nq, seed=n)
    ix = ctx_tc.create_index(f"tcraw_{n}_{d}", d)
    try:
        ix.add(np.arange(n, dtype=np.uint64), x)
        # the pass the search runs: the default one dumps the bf16 pass on split rows, the TF32 mode the TF32 pass
        split = ix.stats().dim_padded % 64 == 0
        tc_pass = _native.TC_PASS_BF16_SPLIT if request.node.callspec.params["ctx_tc"] == "cvt" and split else _native.TC_PASS_TF32
        a = ix.debug_tc_dump_pass(q, tc_pass)         # [nq_pad, S]
        xo, qo = passes.operands(x, q, tc_pass, split)
        xn = (x.astype(np.float64) ** 2).sum(1)
        ref = xn[None, :] - 2.0 * (qo.astype(np.float64) @ xo.astype(np.float64).T)
        got = a[:nq, :n].astype(np.float64)
        err = np.abs(got - ref)
        # fp32 accumulation over k K steps (one ulp of the running magnitude each), |x|^2 and the epilogue's rounding
        absref = np.abs(qo.astype(np.float64)) @ np.abs(xo.astype(np.float64)).T
        k = passes.k_steps(d, tc_pass)
        bound = 2.0 * k * 2.0 ** -23 * absref + (d // 128 + 10) * 2.0 ** -24 * xn[None, :] + 2.0 ** -24 * np.abs(got)
        assert (err <= bound).all(), (err / bound).max()
        assert np.isposinf(a[:nq, n:]).all()          # rows past the end never qualify
        assert np.allclose(a[nq:, :n], xn[None, :], rtol=(d // 128 + 10) * 2.0 ** -24, atol=0)   # zero-filled queries
    finally:
        ix.drop()


@pytest.mark.parametrize("batch,P", [(40, 30), (200, 30), (256, 90), (300, 10), (24, 900)])
def test_tc_pipeline_bit_exact(ctx_tc, oracle, batch, P):
    from kaito_b200 import _native
    n, d = 300_000, 128
    x = oracle.synth_dense(n, d, seed=3)
    q = oracle.synth_queries(x, batch, seed=batch)
    ix = ctx_tc.create_index(f"tc_{batch}_{P}", d)
    try:
        ix.add(np.arange(n, dtype=np.uint64), x)
        fb0 = _native.load().krag_tc_fallback_queries()
        dist, ordn = ix.search_dense(q, P)
        fb = _native.load().krag_tc_fallback_queries() - fb0
        rd, ro = oracle.dense_topk(x, q, P)
        assert np.array_equal(ordn, ro)
        assert np.array_equal(dist, rd)               # exact fp32 rescoring: bit-identical to K1 / oracle
        assert fb <= batch // 20, f"{fb} of {batch} queries needed the exact-scan fallback on random data"
    finally:
        ix.drop()


def test_tc_certificate_fallback_on_adversarial_data(ctx_tc, oracle):
    """6000 near-duplicates of one row overflow a query's candidate list: the certificate must
    fail and the exact scan must still return the right answer; tombstones are honoured."""
    from kaito_b200 import _native
    n, d = 280_000, 64
    x = oracle.synth_dense(n, d, seed=9)
    g = np.random.default_rng(1)
    dup = g.choice(n, 6000, replace=False)
    x[dup] = x[dup[0]] + 1e-4 * g.standard_normal((6000, d)).astype(np.float32)
    q = np.concatenate([x[dup[:1]], oracle.synth_queries(x, 31, seed=4)])
    ix = ctx_tc.create_index("tc_adv", d)
    try:
        ix.add(np.arange(n, dtype=np.uint64), x)
        ix.remove(np.array([int(dup[1]), int(dup[2])], np.uint64))
        alive = oracle.alive_bitmap(n, [int(dup[1]), int(dup[2])])
        fb0 = _native.load().krag_tc_fallback_queries()
        dist, ordn = ix.search_dense(q, 30)
        fb = _native.load().krag_tc_fallback_queries() - fb0
        rd, ro = oracle.dense_topk(x, q, 30, alive)
        assert np.array_equal(ordn, ro) and np.array_equal(dist, rd)
        assert fb >= 1
    finally:
        ix.drop()


@pytest.fixture(scope="module")
def ctx_bf16():
    from kaito_b200 import _native
    c = _native.Context(device_id=0, dense_mode=_native.DENSE_TC_BF16)
    yield c
    c.close()


@pytest.mark.parametrize("batch,P", [(64, 30), (256, 30), (32, 300)])
def test_bf16_shadow_pruning_still_returns_exact_fp32(ctx_bf16, oracle, batch, P):
    """opt-in mode: the tensor-core PRUNE pass reads a bf16 shadow of the corpus; the returned distances are exact
    fp32 re-scores of the fp32 rows and must equal the oracle bit for bit; appends keep the shadow in sync"""
    from kaito_b200 import _native
    n, d = 300_000, 128
    x = oracle.synth_dense(n, d, seed=5)
    q = oracle.synth_queries(x, batch, seed=batch + 1)
    ix = ctx_bf16.create_index(f"bf16_{batch}_{P}", d)
    try:
        ix.add(np.arange(200_000, dtype=np.uint64), x[:200_000])
        ix.add(np.arange(200_000, n, dtype=np.uint64), x[200_000:])
        fb0 = _native.load().krag_tc_fallback_queries()
        dist, ordn = ix.search_dense(q, P)
        fb = _native.load().krag_tc_fallback_queries() - fb0
        rd, ro = oracle.dense_topk(x, q, P)
        assert np.array_equal(ordn, ro) and np.array_equal(dist, rd)
        assert fb <= max(1, batch // 10), fb
        assert _native.last_dense_kernel()[1] == 4      # the bf16-shadow prune pass really ran
    finally:
        ix.drop()


def test_dense_mode_switch_builds_shadow_on_demand(oracle):
    """krag_index_set_dense_mode: AUTO (TF32 over fp32) -> TC_BF16 builds the shadow from the resident rows, later appends
    keep it in sync, switching back releases it; the results are bit-identical in every mode."""
    from kaito_b200 import _native
    n, d, batch, P = 300_000, 128, 64, 30
    x = oracle.synth_dense(n, d, seed=8)
    q = oracle.synth_queries(x, batch, seed=9)
    c = _native.Context(device_id=0)
    try:
        ix = c.create_index("switch", d)
        ix.add(np.arange(280_000, dtype=np.uint64), x[:280_000])
        rd, ro = oracle.dense_topk(x[:280_000], q, P)
        d0, o0 = ix.search_dense(q, P)
        assert _native.last_dense_kernel()[1] == 5 and np.array_equal(o0, ro) and np.array_equal(d0, rd)   # default: convert-in-smem pass
        bytes0 = ix.stats().device_bytes
        ix.set_dense_mode(_native.DENSE_TC_BF16)
        assert ix.stats().device_bytes > bytes0
        d1, o1 = ix.search_dense(q, P)
        assert _native.last_dense_kernel()[1] == 4 and np.array_equal(o1, ro) and np.array_equal(d1, rd)
        ix.add(np.arange(280_000, n, dtype=np.uint64), x[280_000:])           # append with the shadow present
        rd2, ro2 = oracle.dense_topk(x, q, P)
        d2, o2 = ix.search_dense(q, P)
        assert _native.last_dense_kernel()[1] == 4 and np.array_equal(o2, ro2) and np.array_equal(d2, rd2)
        ix.set_dense_mode(_native.DENSE_AUTO, release_shadow=True)
        d3, o3 = ix.search_dense(q, P)
        assert _native.last_dense_kernel()[1] == 5 and np.array_equal(o3, ro2) and np.array_equal(d3, rd2)
        ix.drop()
    finally:
        c.close()


# ---------------------------------------------------------------- K2 at the shapes it is benchmarked on
# bench.py runs K2 at d = 768 (24 fp32 / 12 bf16 k-blocks per tile: the staging ring wraps several times per tile and the
# mbarrier phases flip, unlike d = 128) over millions of rows with NQ = 256.  These cases pin the whole pipeline (sample ->
# threshold -> prune on the tensor cores -> exact rescoring -> certificate) bit-exact against the oracle at those shapes, for both
# the default pass (kernel id 5, fp32 rows rounded to bf16 on chip) and the TF32 pass (id 3).
_BIG = {}


def _big_corpus(oracle, n, d, seed):
    """rows generated on the device (krag_synth_fill), read back for the oracle; the oracle's answer for the widest pool is
    computed once per (shape, batch) and shared by both kernel variants"""
    key = (n, d, seed)
    if key not in _BIG:
        from kaito_b200 import _native
        c = _native.Context(device_id=0, dense_mode=_native.DENSE_SCAN)
        ix = c.create_index("big_src", d)
        ix.synth_fill(n, row_base=0, seed=seed, vocab=0)
        x = ix.read_rows(0, n)
        ix.drop(); c.close()
        _BIG[key] = {"x": x}
    return _BIG[key]


@pytest.mark.parametrize("n,d,batch,pools", [(1_000_000, 768, 256, (30, 900)), (1_000_000, 1024, 64, (30,))])
def test_tc_pipeline_bit_exact_at_bench_shapes(ctx_tc, oracle, n, d, batch, pools):
    from kaito_b200 import _native
    ent = _big_corpus(oracle, n, d, seed=77)
    x = ent["x"]
    q = oracle.synth_queries(x, batch, seed=batch + d)
    okey = ("oracle", batch, max(pools))
    if okey not in ent:
        ent[okey] = oracle.dense_topk(x, q, max(pools))
    rd_all, ro_all = ent[okey]
    ix = ctx_tc.create_index(f"tcbig_{d}_{batch}", d)
    try:
        ix.synth_fill(n, row_base=0, seed=77, vocab=0)
        for P in pools:
            fb0 = _native.load().krag_tc_fallback_queries()
            dist, ordn = ix.search_dense(q, P)
            fb = _native.load().krag_tc_fallback_queries() - fb0
            kid = _native.last_dense_kernel()[1]
            assert kid in (3, 5), kid                                   # the prune pass that bench.py times
            assert np.array_equal(ordn, ro_all[:, :P]), f"ids differ at P={P} (kernel {kid})"
            assert np.array_equal(dist, rd_all[:, :P]), f"distances differ at P={P} (kernel {kid})"
            assert fb <= batch // 20, f"{fb} of {batch} queries fell back to the exact scan on random data"
    finally:
        ix.drop()


def test_tc_adversarial_duplicates_at_d768(ctx_tc, oracle):
    """5000 near-duplicates of one row at d = 768: the query that hits them overflows its candidate list, the certificate
    must fail for it and the exact scan must still return the oracle's answer; everything else stays on the tensor cores"""
    from kaito_b200 import _native
    n, d = 400_000, 768
    ent = _big_corpus(oracle, 1_000_000, 768, seed=77)
    x = ent["x"][:n].copy()
    g = np.random.default_rng(5)
    dup = g.choice(n, 5000, replace=False)
    x[dup] = x[dup[0]] + 1e-5 * g.standard_normal((5000, d)).astype(np.float32)
    q = np.concatenate([x[dup[:1]], oracle.synth_queries(x, 63, seed=6)])
    ix = ctx_tc.create_index("tc_adv768", d)
    try:
        ix.add(np.arange(n, dtype=np.uint64), x)
        fb0 = _native.load().krag_tc_fallback_queries()
        dist, ordn = ix.search_dense(q, 30)
        fb = _native.load().krag_tc_fallback_queries() - fb0
        rd, ro = oracle.dense_topk(x, q, 30)
        assert np.array_equal(ordn, ro) and np.array_equal(dist, rd)
        assert 1 <= fb <= 8, fb
    finally:
        ix.drop()
