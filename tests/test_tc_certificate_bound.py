"""CPU check of the adversarial corpus that tests K2's exactness certificate (test_gpu_dense_edges.py).

K2 (dense_tc.cu) prunes with reduced-precision dot products and certifies a query when
    D_P <= thr + |q|^2 - 2 eps - slack,   eps = eps_rel |x|_max |q|,
where D_P is the P-th exact distance among the admitted rows and thr the per-query threshold of the sample pass.
The certificate is sound only if eps_rel bounds the main pass's dot-product error.  With both operands rounded to
nearest bf16 (8 significant bits) that error reaches 2 * 2^-8 relative, so eps_rel must be at least 2^-7.

adversarial_corpus() builds a corpus on which the kernel's own rounding prunes the true nearest row of one query while
a certificate with a too small eps_rel still passes.  This file emulates that rounding with numpy and checks the
construction, so the GPU test keeps its teeth if the constants of the kernel are retuned.
"""
import numpy as np
import pytest

# kernel constants (dense_tc.cu)
TC_TILE_M, TC_SAMPLE_STRIDE, TC_DUMP_GROUP, TC_MIN_ROWS = 128, 64, 16, 262144
EPS_TF32 = 2.0 ** -9 + 2.0 ** -12               # both operands truncated to TF32
EPS_BF16 = 2.0 ** -7 + 2.0 ** -12               # both operands rounded to nearest bf16
EPS_BF16_HALF = 2.0 ** -8 + 2.0 ** -9 + 2.0 ** -11   # the bf16 bound before it was corrected: half the operand error

N, D = TC_MIN_ROWS, 64
C = np.float32(1.0 + 2.0 ** -8 - 2.0 ** -20)    # just below the bf16 midpoint 1 + 2^-8: rounds down to 1.0 by ~2^-8
TARGET_ROW = 5 * TC_TILE_M + 37                 # outside the sampled tiles (tiles 0, 64, 128, ...)


def bf16_rn(x):
    """fp32 -> bf16 (round to nearest even) -> fp32, as __floats2bfloat162_rn"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def tf32_trunc(x):
    """fp32 -> TF32 as the tensor cores read an fp32 operand: the low 13 mantissa bits are dropped"""
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def sampled_rows(n):
    """rows the sample pass reads: tiles t = 0, 64, 128, ... of 128 rows"""
    t = np.arange(0, (n + TC_TILE_M - 1) // TC_TILE_M, TC_SAMPLE_STRIDE)
    r = (t[:, None] * TC_TILE_M + np.arange(TC_TILE_M)[None, :]).reshape(-1)
    return r[r < n]


def tc_target(P, bf16):
    c, lo = (6 if bf16 else 4) * P, (1024 if bf16 else 512)
    return min(max(c, lo), 3072)


def adversarial_corpus(P):
    """(x [N, D] fp32, q [D] fp32, decoy rows): q = C * ones and its copy x* = row TARGET_ROW.

    - one row per 16-row group of the sampled tiles has a = |x|^2 - 2 x.q = T (ones, three 0.5 and 0.7109375: exact
      in bf16 and TF32), so every group minimum of the sample pass, and with it thr, is T;
    - x* rounds to ones in bf16 while q rounds to ones too: its main-pass a is ~2^-6 |x||q| above its exact a and
      lands at or above thr, so the main pass prunes it although it is the exact nearest row (distance 0);
    - P decoys, exact in bf16 (ones, the k-th with k components at 1 - 2^-8), are admitted and set D_P just above 0;
    - every other row is a random unit vector: far from q, and |x|_max stays |x*|."""
    g = np.random.default_rng(12)
    x = g.standard_normal((N, D), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True).astype(np.float32)
    srow = np.ones(D, np.float32)
    srow[:4] = (0.5, 0.5, 0.5, 0.7109375)
    samp = sampled_rows(N)
    x[samp[::TC_DUMP_GROUP]] = srow
    x[TARGET_ROW] = C
    decoys = np.array([(11 + 3 * k) * TC_TILE_M + 5 * k + 1 for k in range(P)])
    assert not np.isin(decoys, samp).any() and TARGET_ROW not in decoys
    for k, r in enumerate(decoys):
        x[r] = 1.0
        x[r, :k] = np.float32(1.0 - 2.0 ** -8)
    q = np.full(D, C, np.float32)
    return x, q, decoys


def emulate_k2(x, q, P, bf16):
    """numpy model of K2 for one query: (pruned exact nearest row?, certificate inputs).

    Sample pass: TF32 operands; main pass: bf16 (round to nearest) or TF32 operands; products summed in fp64 (the
    tensor cores' fp32 accumulation adds ~1e-6 relative, far inside every margin below)."""
    xn = (x.astype(np.float64) ** 2).sum(1).astype(np.float32).astype(np.float64)
    samp = sampled_rows(x.shape[0])
    a_s = xn[samp] - 2.0 * (tf32_trunc(x[samp]).astype(np.float64) @ tf32_trunc(q).astype(np.float64))
    gmin = a_s.reshape(-1, TC_DUMP_GROUP).min(1)
    m = int(tc_target(P, bf16) * len(samp) / x.shape[0] + 0.5)
    m = min(max(m, 4), 1024, len(gmin))
    thr = np.sort(gmin)[m - 1]
    rnd = bf16_rn if bf16 else tf32_trunc
    a_main = xn - 2.0 * (rnd(x).astype(np.float64) @ rnd(q).astype(np.float64))
    cand = np.nonzero(a_main < thr)[0]
    exact = ((x.astype(np.float64) - q.astype(np.float64)) ** 2).sum(1)
    nearest = int(np.argmin(exact))
    dP = np.sort(exact[cand])[P - 1] if len(cand) >= P else np.inf
    return {"thr": thr, "cand": cand, "nearest": nearest, "pruned": nearest not in set(cand.tolist()),
            "dP": dP, "qn": float((q.astype(np.float64) ** 2).sum()), "xmax": float(xn.max())}


def certified(e, eps_rel):
    eps = eps_rel * np.sqrt(e["xmax"]) * np.sqrt(e["qn"])
    slack = 4e-6 * (1.0 + e["qn"] + e["xmax"])
    return e["dP"] <= e["thr"] + e["qn"] - 2.0 * eps - slack


@pytest.fixture(scope="module", params=[1, 10])
def construction(request):
    P = request.param
    x, q, decoys = adversarial_corpus(P)
    return P, x, q, decoys


def test_rounding_helpers():
    v = np.array([1.0, C, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -C, 0.5], np.float32)
    assert bf16_rn(v).tolist() == [1.0, 1.0, 1.0, 1.0 + 2.0 ** -6, -1.0, 0.5]   # ties to even
    assert tf32_trunc(v).tolist() == [1.0, 1.0 + 3 * 2.0 ** -10, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 3 * 2.0 ** -10), 0.5]


def test_bf16_operand_error_reaches_twice_the_old_bound(construction):
    """x* and q both round down by ~2^-8: the main-pass dot product is off by ~2^-7 |x||q|, above the old bound"""
    P, x, q, _ = construction
    xs = x[TARGET_ROW].astype(np.float64)
    err = (xs @ q.astype(np.float64) - bf16_rn(x[TARGET_ROW]).astype(np.float64) @ bf16_rn(q).astype(np.float64))
    rel = err / (np.linalg.norm(xs) * np.linalg.norm(q.astype(np.float64)))
    assert EPS_BF16_HALF < rel <= EPS_BF16
    assert rel > 0.99 * 2.0 ** -7


def test_construction_prunes_the_nearest_row_and_passes_the_old_certificate(construction):
    """bf16 main pass (TC_CVT and TC_BF16): the exact nearest row is pruned, yet the old bound certifies the query,
    i.e. the old code would return a wrong top P marked as exact; the corrected bound refuses it"""
    P, x, q, decoys = construction
    e = emulate_k2(x, q, P, bf16=True)
    assert e["nearest"] == TARGET_ROW and e["pruned"]
    assert set(decoys.tolist()) <= set(e["cand"].tolist()) and len(e["cand"]) < 4 * tc_target(P, True)
    assert certified(e, EPS_BF16_HALF), "the construction no longer fools the old bf16 bound"
    assert not certified(e, EPS_BF16), "the corrected bf16 bound must not certify this query"


def threshold_window(x, q, P):
    """(lo, hi): a threshold thr with lo < thr < hi prunes x* in a bf16 main pass while the old bound still certifies
    the query (hi: main-pass a of x*; lo: D_P - |q|^2 + 2 eps_old + slack)"""
    e = emulate_k2(x, q, P, bf16=True)
    xs = x[TARGET_ROW].astype(np.float64)
    xn = float(np.float32((xs ** 2).sum()))
    hi = xn - 2.0 * float(bf16_rn(x[TARGET_ROW]).astype(np.float64) @ bf16_rn(q).astype(np.float64))
    eps_old = EPS_BF16_HALF * np.sqrt(e["xmax"] * e["qn"])
    lo = e["dP"] - e["qn"] + 2.0 * eps_old + 4e-6 * (1.0 + e["qn"] + e["xmax"])
    return lo, hi


def test_construction_margins_cover_tf32_rounding_mode(construction):
    """the threshold lies inside the window with room to spare, also if the sample pass rounded its operands to
    nearest instead of truncating them (the threshold then moves down by ~0.12)"""
    P, x, q, _ = construction
    e = emulate_k2(x, q, P, bf16=True)
    lo, hi = threshold_window(x, q, P)
    srow = x[sampled_rows(N)[0]].astype(np.float64)
    q_rn = (q.view(np.uint32).astype(np.uint64) + 0x1000) & 0xFFFFE000
    thr_rn = float(np.float32((srow ** 2).sum())) - 2.0 * srow @ q_rn.astype(np.uint32).view(np.float32).astype(np.float64)
    for thr in (e["thr"], thr_rn):
        assert lo + 0.02 < thr < hi - 0.02, (lo, thr, hi)


def test_tf32_main_pass_admits_the_nearest_row(construction):
    """TC_TF32: the truncation error is small enough that x* is admitted and the certificate holds honestly"""
    P, x, q, _ = construction
    e = emulate_k2(x, q, P, bf16=False)
    assert not e["pruned"]
    assert certified(e, EPS_TF32)
