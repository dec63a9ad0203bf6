"""The bf16 copy of an index's dense rows covers every row, whichever index of the context switched the mode.

krag_index_set_dense_mode sets the dense mode of the whole context.  An index that already holds rows when another index
of its context switches to KRAG_DENSE_TC_BF16 gets its bf16 shadow on its next add or reserve; the shadow must then be
built from the rows it already has, not only from the rows that add brings.  K2's exactness certificate assumes the
shadow is bf16(x) for every row, so a stale row there can certify a wrong top P."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

D = 768
N_FIRST = 150_000
N_TOTAL = 300_000          # above TC_MIN_ROWS (262,144): the batch below runs K2
NQ, K = 64, 10


@pytest.mark.parametrize("grow", ["add", "reserve"])
def test_shadow_from_another_index_covers_the_old_rows(grow):
    from kaito_b200 import _native as N
    rng = np.random.default_rng(7)
    x = rng.standard_normal((N_TOTAL, D), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    planted = np.arange(0, N_FIRST, N_FIRST // NQ)[:NQ]                    # queries next to rows of the first add
    q = (x[planted] + 0.05 * rng.standard_normal((NQ, D), dtype=np.float32)).astype(np.float32)
    c = N.Context(device_id=0)
    try:
        a = c.create_index("a", D)
        b = c.create_index("b", D)
        a.add(np.arange(N_FIRST, dtype=np.uint64), x[:N_FIRST])            # no shadow yet (KRAG_DENSE_AUTO)
        b.set_dense_mode(N.DENSE_TC_BF16)                                  # the context's mode, set through b
        if grow == "reserve":
            a.reserve(N_TOTAL)
        a.add(np.arange(N_FIRST, N_TOTAL, dtype=np.uint64), x[N_FIRST:])
        fallbacks = N.load().krag_tc_fallback_queries()
        dist, ordn = a.search_dense(q, K)
        assert N.last_dense_kernel()[1] == 4, "the batch must prune on the bf16 shadow"
        assert N.load().krag_tc_fallback_queries() == fallbacks, "every query must be certified on the shadow, not re-run on K1"
        b.set_dense_mode(N.DENSE_SCAN)
        ref_dist, ref_ord = a.search_dense(q, K)
        assert N.last_dense_kernel()[1] == 1
        assert np.array_equal(ref_ord[:, 0], planted), "every query's nearest row is the one it was planted next to"
        assert np.array_equal(ordn, ref_ord) and np.array_equal(dist.view(np.uint32), ref_dist.view(np.uint32))
        a.drop()
        b.drop()
    finally:
        c.close()
