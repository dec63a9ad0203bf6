"""KRAG_ROWS_HOST on the GPU: fp32 rows in pinned host memory, a bf16 copy on the device.  Every search must return what
device-resident rows return (K1's exact fp32 distances, ties by ordinal), compared with array_equal: on the K2 path (sample +
main pass on the bf16 rows, refine, fetch, zero-copy rescoring), through its certificate fallback, and on the streamed exact
scan.  Pinned memory stays below ~4 GB at any time."""
import numpy as np
import pytest

from tests import test_host_rows_bound as bound
from tests import test_tc_certificate_bound as adv

pytestmark = pytest.mark.gpu


def _N():
    from kaito_b200 import _native
    return _native


def _fallbacks():
    return _N().load().krag_tc_fallback_queries()


def _same(got, ref, what):
    (gd, go), (rd, ro) = got, ref
    assert np.array_equal(go, ro), f"{what}: ids differ (first bad query {np.nonzero((go != ro).any(1))[0][:5]})"
    assert np.array_equal(gd, rd), f"{what}: distances differ"


@pytest.fixture(scope="module")
def pair():
    """one device-rows and one host-rows context"""
    N = _N()
    dev, host = N.Context(device_id=0), N.Context(device_id=0, row_storage=N.ROWS_HOST)
    yield dev, host
    host.close()
    dev.close()


# --------------------------------------------------------------------------- 1M x 768: K2 over host rows
ROWS, DIM = 1 << 20, 768


@pytest.fixture(scope="module")
def big(pair):
    dev, host = pair
    a, b = dev.create_index("hr_big_dev", DIM), host.create_index("hr_big_host", DIM)
    a.synth_fill(ROWS, 0, 11)
    b.synth_fill(ROWS, 0, 11)
    g = np.random.default_rng(5)
    seeds = a.read_rows(0, 4096)[g.integers(0, 4096, 257)]
    q = (seeds + 0.1 * g.standard_normal(seeds.shape) / np.sqrt(DIM)).astype(np.float32)
    yield a, b, q
    b.drop()
    a.drop()


def test_host_fill_matches_device_fill(big):
    a, b, _ = big
    for r0 in (0, ROWS // 2 + 7, ROWS - 33):
        assert np.array_equal(a.read_rows(r0, 33), b.read_rows(r0, 33))
    sa, sb = a.stats(), b.stats()
    assert sb.device_bytes < sa.device_bytes * 0.55   # bf16 rows + xnorm + xres against fp32 rows + xnorm


@pytest.mark.parametrize("P", [1, 30, 900, 1024])
@pytest.mark.parametrize("batch", [1, 15, 16, 64, 256, 257])
def test_host_k2_equals_device(big, batch, P):
    N = _N()
    a, b, q = big
    ref = a.search_dense(q[:batch], P)
    fb0, f0 = _fallbacks(), N.host_rows_fetched()
    got = b.search_dense(q[:batch], P)
    fb, fetched = _fallbacks() - fb0, N.host_rows_fetched() - f0
    _same(got, ref, f"batch={batch} P={P}")
    kid = N.last_dense_kernel()[1]
    assert kid == 6 or (kid == 1 and fb > 0), (kid, fb)
    # fetched rows: at least P per query, fewer than the main pass's candidate target per query
    assert batch * P <= fetched < batch * adv.tc_target(P, True), (fetched, batch, P)


# --------------------------------------------------------------------------- certificate fallback and the refine bound
def host_adversarial_corpus(P):
    """test_tc_certificate_bound's corpus for a bf16 SAMPLE pass: with host rows the sample pass also reads the bf16 copy,
    where q = C * ones rounds to ones instead of TF32's 1 + 3 * 2^-10, which lifts thr above the window that prunes x*.
    Threshold rows of ones with 0.5 and 0.59375 (exact in bf16) put the bf16 sample value back inside it."""
    x, q, _ = adv.adversarial_corpus(P)
    srow = np.ones(adv.D, np.float32)
    srow[:2] = (0.5, 0.59375)
    x[adv.sampled_rows(adv.N)[::adv.TC_DUMP_GROUP]] = srow
    lo, hi = adv.threshold_window(x, q, P)
    thr = float(np.float32((srow.astype(np.float64) ** 2).sum())) - 2.0 * float(srow.astype(np.float64) @ adv.bf16_rn(q))
    assert lo + 0.05 < thr < hi - 0.05, (lo, thr, hi)
    return x, q


@pytest.mark.parametrize("P", [1, 10])
def test_adversarial_certificate_corpus(pair, oracle, P):
    """the bf16 main pass prunes the exact nearest row: the certificate fails and the streamed scan answers"""
    dev, host = pair
    x, q_adv = host_adversarial_corpus(P)
    q = np.concatenate([q_adv[None, :], oracle.synth_queries(x, 15, seed=40 + P)])
    ref = oracle.dense_topk(x, q, P)
    assert ref[1][0, 0] == adv.TARGET_ROW
    ix = host.create_index(f"hr_adv_{P}", adv.D)
    try:
        ix.add(np.arange(adv.N, dtype=np.uint64), x)
        fb0 = _fallbacks()
        got = ix.search_dense(q, P)
        assert _fallbacks() - fb0 >= 1
        _same(got, ref, f"adversarial P={P}")
    finally:
        ix.drop()


@pytest.mark.parametrize("P", [1, 10])
def test_bf16_inversion_corpus(pair, P):
    """the bf16 copies reverse the true P-th and (P+1)-th rows; the refine bound keeps the true one"""
    N = _N()
    dev, host = pair
    x, q, a_row, _ = bound.inversion_corpus(P)
    qs = np.repeat(q[None, :], 3, 0)
    a, b = dev.create_index(f"hr_inv_dev_{P}", bound.INV_D), host.create_index(f"hr_inv_host_{P}", bound.INV_D)
    try:
        a.add(np.arange(bound.INV_N, dtype=np.uint64), x)
        b.add(np.arange(bound.INV_N, dtype=np.uint64), x)
        fb0 = _fallbacks()
        got = b.search_dense(qs, P)
        assert _fallbacks() == fb0 and N.last_dense_kernel()[1] == 6
        _same(got, a.search_dense(qs, P), f"inversion P={P}")
        assert (got[1][:, P - 1] == a_row).all()
    finally:
        b.drop()
        a.drop()


# --------------------------------------------------------------------------- streamed exact scan
@pytest.mark.parametrize("n,dim", [(300_000, 800), (200_000, 33), (1000, 96)])
def test_streamed_scan(pair, n, dim):
    """dims whose padded width is not a multiple of 64, indexes below the K2 size and small indexes: chunks of host rows
    through K1, tombstones on both sides of every chunk boundary"""
    N = _N()
    dev, host = pair
    g = np.random.default_rng(n + dim)
    x = g.standard_normal((n, dim)).astype(np.float32)
    a, b = dev.create_index(f"hr_scan_dev_{n}_{dim}", dim), host.create_index(f"hr_scan_host_{n}_{dim}", dim)
    try:
        ids = np.arange(n, dtype=np.uint64)
        a.add(ids, x)
        b.add(ids, x)
        dpad = (dim + 31) // 32 * 32
        R = min((64 << 20) // (dpad * 4), 65536) // 32 * 32
        bounds = np.arange(R, n, R)
        assert n < R or (len(bounds) >= 3 and n % R != 0)
        dead = np.unique(np.clip(np.concatenate([bounds - 1, bounds, bounds + 1, [3, n - 1]]), 0, n - 1)).astype(np.uint64)
        assert a.remove(dead) == b.remove(dead) == len(dead)
        q = np.concatenate([x[dead[:8].astype(np.int64)], x[g.integers(0, n, 12)] + 0.01]).astype(np.float32)
        for P in (1, 100):
            got = b.search_dense(q, P)
            assert N.last_dense_kernel()[1] == 1
            _same(got, a.search_dense(q, P), f"scan n={n} dim={dim} P={P}")
    finally:
        b.drop()
        a.drop()


# --------------------------------------------------------------------------- filters, ordinal maps, hybrid retrieve
@pytest.fixture(scope="module")
def hybrid(pair):
    dev, host = pair
    n, dim, vocab = 300_000, 128, 20_000
    a, b = dev.create_index("hr_hyb_dev", dim), host.create_index("hr_hyb_host", dim)
    a.synth_fill(n, 0, 21, vocab)
    b.synth_fill(n, 0, 21, vocab)
    for ix in (a, b):
        ix.remove(np.arange(5, n, 97, dtype=np.uint64))
        ix.commit(vocab)
    g = np.random.default_rng(8)
    q = (a.read_rows(0, 300)[:64] + 0.05 * g.standard_normal((64, dim))).astype(np.float32)
    terms = [list(g.integers(0, 200, g.integers(1, 6))) for _ in range(64)]
    yield a, b, q, terms, n
    b.drop()
    a.drop()


def test_hybrid_retrieve_equals_device(hybrid):
    a, b, q, terms, n = hybrid
    for batch in (1, 64):
        ra, rb = a.retrieve(q[:batch], terms[:batch], 10), b.retrieve(q[:batch], terms[:batch], 10)
        for key in ra:
            assert np.array_equal(ra[key], rb[key], equal_nan=True), (batch, key)


def test_filter_pushdown_and_tombstones(hybrid):
    N = _N()
    a, b, q, terms, n = hybrid
    g = np.random.default_rng(9)
    allow = g.integers(0, 2 ** 32, (n + 31) // 32, dtype=np.uint64).astype(np.uint32)
    for qt in (terms, None):
        kw = dict(fusion_mode=N.FUSION_REFERENCE | N.FILTER_PUSHDOWN, keyword_allow_bitmap=allow)
        ra, rb = a.retrieve(q, qt, 20, **kw), b.retrieve(q, qt, 20, **kw)
        for key in ra:
            assert np.array_equal(ra[key], rb[key], equal_nan=True), key
    _same(b.search_dense(q, 50), a.search_dense(q, 50), "tombstones")


def test_ordinal_map(pair):
    dev, host = pair
    n, dim = 270_000, 64
    g = np.random.default_rng(4)
    x = g.standard_normal((n, dim)).astype(np.float32)
    a, b = dev.create_index("hr_ord_dev", dim), host.create_index("hr_ord_host", dim)
    try:
        for ix in (a, b):
            ix.add(np.arange(n, dtype=np.uint64), x)
            ix.set_ordinal_map(1, 2)
            ix.remove(np.arange(0, n, 13, dtype=np.uint64))
        q = (x[:40] + 0.01).astype(np.float32)
        got = b.search_dense(q, 30)
        _same(got, a.search_dense(q, 30), "ordinal map")
        assert (got[1] % 2 == 1).all()
    finally:
        b.drop()
        a.drop()


# --------------------------------------------------------------------------- life cycle
def test_life_cycle(tmp_path):
    N = _N()
    dev0, pin0 = N.device_bytes(), N.host_pinned_bytes()
    dev, host = N.Context(device_id=0), N.Context(device_id=0, row_storage=N.ROWS_HOST)
    try:
        n, dim = 300_000, 192
        g = np.random.default_rng(1)
        x = g.standard_normal((n, dim)).astype(np.float32)
        b = host.create_index("hr_life", dim)
        caps = []
        for lo, hi in ((0, 1000), (1000, 40_000), (40_000, n)):   # three adds, each growing the pinned rows
            b.add(np.arange(lo, hi, dtype=np.uint64), x[lo:hi])
            caps.append(N.host_pinned_bytes())
        assert caps[0] < caps[1] < caps[2] and caps[2] >= pin0 + n * dim * 4
        assert np.array_equal(b.read_rows(0, n), x)
        q = (x[g.integers(0, n, 32)] + 0.02).astype(np.float32)
        ref = b.search_dense(q, 40)
        b.persist(str(tmp_path / "h"))
        a = dev.load_index("hr_life_dev", str(tmp_path / "h"))           # host-mode snapshot into device rows
        _same(a.search_dense(q, 40), ref, "host snapshot in device mode")
        a.persist(str(tmp_path / "d"))
        b2 =host.load_index("hr_life_2", str(tmp_path / "d"))           # and back
        _same(b2.search_dense(q, 40), ref, "device snapshot in host mode")
        assert np.array_equal(b2.read_rows(0, n), x)
        b2.set_dense_mode(N.DENSE_SCAN)
        _same(b2.search_dense(q, 40), ref, "scan mode")
        assert N.last_dense_kernel()[1] == 1
        b2.set_dense_mode(N.DENSE_TC_BF16, release_shadow=True)
        _same(b2.search_dense(q, 40), ref, "TC_BF16 after release_shadow")
        b2.set_dense_mode(N.DENSE_AUTO, release_shadow=True)             # the bf16 rows are the index's device copy: kept
        _same(b2.search_dense(q, 40), ref, "AUTO after release_shadow")
        with pytest.raises(N.KragError) as e:
            b2.debug_tc_dump(q[:1])
        assert e.value.code == N.KRAG_E_UNSUPPORTED
        for ix in (b2, a, b):
            ix.drop()
        assert N.host_pinned_bytes() == pin0
    finally:
        host.close()
        dev.close()
    assert N.device_bytes() == dev0 and N.host_pinned_bytes() == pin0


# --------------------------------------------------------------------------- service
def test_service_host_rows_equals_device(tmp_path):
    from starlette.testclient import TestClient

    from kaito_b200.embedding import HashingEmbedding
    from kaito_b200.service import create_app
    from kaito_b200.vector_store import VectorStore
    from tests.test_service import CFG, _exercise
    N = _N()
    out = []
    for storage in ("device", "host"):
        c = N.Context(device_id=0, row_storage=N.row_storage_from_env({"KRAG_ROW_STORAGE": storage}))
        try:
            out.append(_exercise(TestClient(create_app(VectorStore(HashingEmbedding(64), c), dict(CFG))), tmp_path))
        finally:
            c.close()
    assert out[0] == out[1]
