"""K2's bf16 prune pass on 192-row tiles (dense_tc_bf16_kernel) value by value against fp64.

Each tile is three 64-row blocks: warpgroup w multiplies rows 64 w .. 64 w + 63 by every query of the NQ bucket, and
rows 128 .. 191 by queries w NQ/2 .. w NQ/2 + NQ/2 - 1, so the upper half of a bucket's queries is computed by the
second warpgroup only.  The shapes cover every tile tail that changes which blocks hold real rows (n % 192 in {0, 1, 63,
64, 65, 127, 128, 129, 191}) and batches on both sides of every bucket edge (64 / 65, 128 / 129, 255 / 256).  All three
bf16 passes are checked through krag_debug_tc_dump_pass against the bound of test_gpu_tc_passes.py, and
krag_debug_tc_prune's candidate lists against the dump, with tombstones; searches at 1M x 768 with a batch of 256 must
equal the exact scan (K1).
"""
import numpy as np
import pytest

from tests import test_gpu_tc_passes as passes

pytestmark = pytest.mark.gpu

TAILS = [0, 1, 63, 64, 65, 127, 128, 129, 191]
BATCHES = [65, 129, 255, 64, 128, 256, 1, 200, 100]       # one per tail: every bucket, full and padded


def _native():
    from kaito_b200 import _native
    return _native


@pytest.fixture(scope="module")
def ctx_bf16():
    N = _native()
    c = N.Context(device_id=0, dense_mode=N.DENSE_TC_BF16)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx_host():
    N = _native()
    c = N.Context(device_id=0, row_storage=N.ROWS_HOST)
    yield c
    c.close()


@pytest.mark.parametrize("tail,nq", list(zip(TAILS, BATCHES)))
def test_bf16_passes_at_every_tile_tail(ctx_bf16, ctx_host, oracle, tail, nq):
    """two full tiles and a tail: split high halves, shadow and host copy against fp64 over their own operands"""
    N = _native()
    n, dpad = 2 * 192 + tail, 128 if tail % 2 else 768
    x = oracle.synth_dense(n, dpad, seed=tail + 1)
    q = oracle.synth_queries(x, nq, seed=nq)
    ix, hx = passes._index(ctx_bf16, f"t192_{tail}", x), passes._index(ctx_host, f"t192h_{tail}", x)
    try:
        for p in (N.TC_PASS_BF16_SPLIT, N.TC_PASS_BF16_SHADOW):
            passes.check_pass(ix, x, q, p, what=f"tail {tail}")
        passes.check_pass(hx, x, q, N.TC_PASS_BF16_HOST, what=f"tail {tail}")
    finally:
        hx.drop()
        ix.drop()


@pytest.mark.parametrize("nq", [65, 129, 255])
def test_bf16_passes_exact_on_integer_data(ctx_bf16, ctx_host, nq):
    """integer rows and queries: every product and partial sum is exact, so each pass must equal fp64 bit for bit in
    every block of the tile, padded query columns included"""
    N = _native()
    n, dpad = 3 * 192 + 129, 256
    x = passes.integer_rows(n, dpad, seed=nq)
    q = passes.integer_rows(nq, dpad, seed=nq + 1)
    ix, hx = passes._index(ctx_bf16, f"t192i_{nq}", x), passes._index(ctx_host, f"t192ih_{nq}", x)
    try:
        for p in (N.TC_PASS_BF16_SPLIT, N.TC_PASS_BF16_SHADOW):
            passes.check_pass(ix, x, q, p, exact=True, what="integer")
        passes.check_pass(hx, x, q, N.TC_PASS_BF16_HOST, exact=True, what="integer")
    finally:
        hx.drop()
        ix.drop()


@pytest.mark.parametrize("nq", [64, 129, 255])
def test_candidate_lists_with_tombstones(ctx_bf16, ctx_host, oracle, nq):
    """krag_debug_tc_prune against the dump on n % 192 = 191 with 10 % tombstones, padded columns admitting everything,
    half the rows or nothing: the lists of every pass are the alive rows below the threshold"""
    N = _native()
    n, dpad = 5 * 192 + 191, 128
    x = oracle.synth_dense(n, dpad, seed=nq + 3)
    q = oracle.synth_queries(x, nq, seed=nq + 4)
    dead = np.random.default_rng(nq).choice(n, n // 10, replace=False)
    alive = np.ones(n, bool)
    alive[dead] = False

    def wide(k, xn):
        t = np.full(k, np.inf, np.float32)
        t[1::3] = np.float32(np.median(xn))
        t[2::3] = -np.inf
        return t

    ix, hx = passes._index(ctx_bf16, f"t192e_{nq}", x), passes._index(ctx_host, f"t192eh_{nq}", x)
    try:
        for index in (ix, hx):
            index.remove(dead.astype(np.uint64))
        for index, p in ((ix, N.TC_PASS_BF16_SPLIT), (ix, N.TC_PASS_BF16_SHADOW), (hx, N.TC_PASS_BF16_HOST)):
            thr, counts, _ = passes._emission(index, x, q, alive, p, wide, f"{passes.PASS_NAMES[p]} nq={nq}")
            if nq < len(thr):
                assert counts[nq] == alive.sum()                      # +inf: every alive row, none past n
            if nq + 2 < len(thr):
                assert counts[nq + 2] == 0                            # -inf: nothing
    finally:
        hx.drop()
        ix.drop()


def test_search_1m_batch256_equals_exact_scan():
    """1M x 768 (5208 full tiles and a 64-row tail) with tombstones, a batch of 256 (one full bucket) and 255: the
    default pass (split high halves), the shadow and the host copy return exactly what K1 returns"""
    N = _native()
    n, dim, P = 1_000_000, 768, 30
    dev, host = N.Context(device_id=0), N.Context(device_id=0, row_storage=N.ROWS_HOST)
    a, b = dev.create_index("t192_1m", dim), host.create_index("t192_1m_host", dim)
    try:
        a.synth_fill(n, 0, 17)
        b.synth_fill(n, 0, 17)
        dead = np.arange(3, n, 211, dtype=np.uint64)
        assert a.remove(dead) == len(dead) and b.remove(dead) == len(dead)
        g = np.random.default_rng(19)
        seeds = a.read_rows(0, 8192)[g.integers(0, 8192, 256)]
        q = (seeds + 0.1 * g.standard_normal(seeds.shape) / np.sqrt(dim)).astype(np.float32)
        a.set_dense_mode(N.DENSE_SCAN)
        ref = {batch: a.search_dense(q[:batch], P) for batch in (256, 255)}
        assert N.last_dense_kernel()[1] == 1
        for index, mode, kid in ((a, N.DENSE_TC, 5), (a, N.DENSE_TC_BF16, 4), (b, None, 6)):
            if mode is not None:
                index.set_dense_mode(mode)
            for batch in (256, 255):
                fb0 = N.load().krag_tc_fallback_queries()
                d, o = index.search_dense(q[:batch], P)
                fb = N.load().krag_tc_fallback_queries() - fb0
                assert N.last_dense_kernel()[1] == kid or (fb > 0 and N.last_dense_kernel()[1] == 1), (kid, fb)
                assert np.array_equal(o, ref[batch][1]), f"kernel {kid} batch {batch}: ids differ"
                assert np.array_equal(d, ref[batch][0]), f"kernel {kid} batch {batch}: distances differ"
    finally:
        b.drop()
        a.drop()
        host.close()
        dev.close()
