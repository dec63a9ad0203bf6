"""CPU restatement of the refine interval and the fetch rule of K2 over host-resident rows (dense_tc.cu: refine_kernel,
fetch_compact_kernel, fetch_rule_constants).

With the fp32 rows x in host memory, the device holds b = bf16(x) and r >= |x - b| (rounded up).  For every candidate the
refine pass bounds the exact distance D = |x - q|^2 by
    L = max(0, sqrt(d_lo) - r)^2 <= D <= U = (sqrt(d_hi) + r)^2,      d_lo <= |b - q|^2 <= d_hi,
rounding every step outwards.  K1 rounds D to D1 with |D1 - D| <= gamma D + eta (gamma = m u / (1 - m u), m = dpad / 32 + 7).
With U_(P) the P-th smallest U, a candidate is fetched iff L <= T = ((1 + gamma) U_(P) + 2 eta) / (1 - gamma); everything
else is strictly worse, after K1's rounding, than P fetched rows.

Here numpy emulates the kernel's directed rounding by computing in float64 and stepping one float32 ulp outwards, and K1's
summation order in float32.  inversion_corpus() builds rows whose bf16 copies swap the true P-th and (P+1)-th nearest rows:
a rule that ignores r drops the true P-th row; the GPU test (test_gpu_host_rows.py) runs it on the kernels.
"""
import numpy as np
import pytest

from tests.test_tc_certificate_bound import bf16_rn

U32 = 2.0 ** -24


def k1_l2sq(x, q):
    """K1's fp32 operation order (dense_scan.cu): lane l of 8 owns elements 32 i + 4 l + c; FFMA chains per c; (p0 + p1) +
    (p2 + p3); butterfly over lanes 4, 2, 1.  FMA emulated in float64 (t * t is exact there)."""
    x = np.atleast_2d(np.asarray(x, np.float32))
    n, dpad = x.shape
    t = (x - np.asarray(q, np.float32)[None, :]).astype(np.float32)
    t = t.reshape(n, dpad // 32, 8, 4).astype(np.float64)
    acc = np.zeros((n, 8, 4), np.float32)
    for i in range(dpad // 32):
        acc = (acc.astype(np.float64) + t[:, i] * t[:, i]).astype(np.float32)
    s = (acc[..., 0] + acc[..., 1]) + (acc[..., 2] + acc[..., 3])
    for o in (4, 2, 1):
        s = s + s[:, np.arange(8) ^ o]
    return s[:, 0]


def down(v):
    return np.nextafter(np.asarray(v, np.float64).astype(np.float32), np.float32(-np.inf))


def up(v):
    return np.nextafter(np.asarray(v, np.float64).astype(np.float32), np.float32(np.inf))


def xres(x):
    """|x - bf16(x)| rounded up (bf16_residual_kernel)"""
    e = (np.asarray(x, np.float32) - bf16_rn(x)).astype(np.float64)
    return up(np.sqrt((e * e).sum(-1)))


def refine_interval(x, q, res=None):
    """(L, U) per row from the bf16 copy and r; res=0 gives the rule without the residual term"""
    b = bf16_rn(x).astype(np.float64)
    d = ((b - np.asarray(q, np.float64)[None, :]) ** 2).sum(-1)
    d_lo, d_hi = np.maximum(down(d), 0.0), up(d)
    r = xres(x).astype(np.float64) if res is None else np.float64(res)
    lo = down(np.maximum(down(np.sqrt(d_lo)) - r, 0.0).astype(np.float64) ** 2)
    hi = up(up(up(np.sqrt(d_hi)).astype(np.float64) + r).astype(np.float64) ** 2)
    return lo.astype(np.float64), hi.astype(np.float64)


def fetch_constants(dpad):
    m = dpad // 32 + 7
    gamma = m * U32 / (1 - m * U32)
    eta = (dpad + 64) * 2.0 ** -149
    return float(up((1 + gamma) / (1 - gamma))), float(up(2 * eta / (1 - gamma))), gamma, eta


def fetched(L, U, P, dpad):
    """the fetch rule over one query's candidates: boolean mask"""
    if len(U) < P:
        return np.ones(len(U), bool)
    scale, eta2, _, _ = fetch_constants(dpad)
    T = float(up(float(up(np.sort(U)[P - 1] * scale)) + eta2))
    return L <= T


def top_p_k1(x, q, P):
    """K1's answer: the P smallest (fp32 value, ordinal)"""
    d = k1_l2sq(x, q)
    return np.lexsort((np.arange(len(d)), d))[:P], d


# -------------------------------------------------------------------------------- bf16 inversion construction
INV_N, INV_D = 262144, 64
C0, ULP = 2.0 ** -5, 2.0 ** -12   # components near 2^-5 and the bf16 spacing there


def inversion_corpus(P, seed=3):
    """(x [N, D] fp32, q [D], row_a, row_b): q = 0; the true P-th nearest row a and (P+1)-th b swap order in bf16.

    - every component of a is C0 + 0.51 ulp: bf16 rounds each up by 0.49 ulp;
    - b has 63 components at C0 + 1.49 ulp (bf16 rounds down by 0.49 ulp) and one at C0 + 0.49 ulp (rounds down to C0):
      |b| > |a| in fp32, |bf16(b)| < |bf16(a)|;
    - P - 1 rows exact in bf16 and nearer than both (components 2^-6 + k 2^-13 in the first place);
    - every other row is a random unit vector (distance ~1, far beyond |a|^2 ~ 1/16)."""
    g = np.random.default_rng(seed)
    x = g.standard_normal((INV_N, INV_D), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True).astype(np.float32)
    row_a, row_b = 9 * 128 + 77, 3 * 128 + 5          # b has the lower ordinal: a tie would also favour it
    x[row_a] = np.float32(C0 + 0.51 * ULP)
    x[row_b] = np.float32(C0 + 1.49 * ULP)
    x[row_b, 17] = np.float32(C0 + 0.49 * ULP)
    for k in range(P - 1):
        r = 20 * 128 + 3 * k
        x[r] = np.float32(2.0 ** -6)
        x[r, 0] = np.float32(2.0 ** -6 + k * 2.0 ** -13)
    return x, np.zeros(INV_D, np.float32), row_a, row_b


# ------------------------------------------------------------------------------------------------------ tests
def _check_rule(x, q, P):
    """the exact distance and K1's value lie in [L, U], and the fetched set contains K1's top P"""
    dpad = x.shape[1]
    L, U = refine_interval(x, q)
    exact = ((x.astype(np.float64) - q.astype(np.float64)[None, :]) ** 2).sum(1)
    top, d1 = top_p_k1(x, q, P)
    _, _, gamma, eta = fetch_constants(dpad)
    assert (L <= exact).all() and (exact <= U).all()
    assert (np.abs(d1 - exact) <= gamma * exact + eta).all()
    keep = fetched(L, U, P, dpad)
    assert keep[top].all(), "a row of K1's top P was not fetched"
    return keep


@pytest.mark.parametrize("P", [1, 10, 30])
def test_rule_on_random_unit_rows(P):
    g = np.random.default_rng(P)
    x = g.standard_normal((3000, 768)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True).astype(np.float32)
    for j in range(4):
        q = (x[j] + 0.3 * g.standard_normal(768) / np.sqrt(768)).astype(np.float32)
        keep = _check_rule(x, q, P)
        assert keep.sum() < len(x) // 4   # the rule is selective on ordinary data


@pytest.mark.parametrize("P", [1, 10])
def test_rule_on_rows_at_bf16_cell_edges(P):
    """components just below / above bf16 midpoints (every element rounds by almost half a bf16 ulp), queries equal to
    rows and to their bf16 copies"""
    g = np.random.default_rng(7 + P)
    base = bf16_rn(g.standard_normal((2000, 128)).astype(np.float32) * 0.1)
    ulp = (base.view(np.uint32) & 0x7F800000).view(np.float32) * 2.0 ** -7
    side = g.choice([-1.0, 1.0], size=base.shape)
    x = (base + side * (0.5 - 2.0 ** -10) * ulp).astype(np.float32)
    for q in (x[0], bf16_rn(x[1]), x[2] + np.float32(1e-3)):
        _check_rule(x, np.asarray(q, np.float32), P)


@pytest.mark.parametrize("P", [1, 10])
def test_bf16_inversion_needs_the_residual_term(P):
    x, q, a, b = inversion_corpus(P)
    top, d1 = top_p_k1(x, q, P)
    assert top[-1] == a and d1[b] > d1[a], "a is the true P-th row, b the (P+1)-th"
    bd = ((bf16_rn(x[[a, b]]).astype(np.float64)) ** 2).sum(1)
    assert bd[1] < bd[0], "bf16 copies reverse the order"
    # candidates: the K2 main pass admits the near rows (far rows are ~1 away); the rule sees the nearest few hundred
    cand = np.argsort(((bf16_rn(x).astype(np.float64)) ** 2).sum(1))[:300]
    L, U = refine_interval(x[cand], q)
    keep = fetched(L, U, P, INV_D)
    assert keep[list(cand).index(a)], "the rule with the residual term fetches the true P-th row"
    L0, U0 = refine_interval(x[cand], q, res=0.0)
    keep0 = fetched(L0, U0, P, INV_D)
    assert not keep0[list(cand).index(a)], "a rule without the residual term drops the true P-th row"
    _check_rule(x[cand], q, P)
