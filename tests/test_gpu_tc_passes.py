"""K2's prune passes value by value against fp64 (krag_debug_tc_dump_pass, krag_debug_tc_prune).

Every pass is checked against an fp64 product of its own operands:
  split rows (BF16_SPLIT)      hi = split_hi(x), bf16 rounded to nearest with ties toward zero; queries bf16 RNE
  shadow, host copy (BF16_*)   bf16 RNE of x; queries bf16 RNE
  TF32 (TC_TF32S, TC_TF32)     x and q truncated to TF32
The dump holds a = fma(-2, acc, xn) per (query, row).  A padded query column of the NQ bucket runs a zero query, so it
returns xn, the row's stored |x|^2, exactly; acc is then rebuilt as (xn - a) / 2, which is within 2^-25 |a| of the fp32
accumulator (a is rounded once).  The accumulator of k tensor-core K steps (K = 16 bf16 or 8 tf32 elements each) is
held to the bound
    |acc - sum hi q^|  <=  k 2^-23 sum |hi q^|
i.e. at most one fp32 ulp of the running magnitude per accumulation step, whatever the hardware's internal order and
rounding.  The bound is derived, not fitted: each test reports the largest error over the bound it saw.

krag_debug_tc_prune runs the non-DUMP main pass with chosen thresholds: its candidate lists must be the rows whose
dumped a is below the threshold, up to a few-ulp band where the epilogue's `acc + thr/2 > xn/2` and the dump's fma round
differently.
"""
import numpy as np
import pytest

from tests.test_split_rows_cpu import split_hi
from tests.test_tc_certificate_bound import EPS_BF16, EPS_TF32, bf16_rn, tf32_trunc

pytestmark = pytest.mark.gpu

KRAG_E_STATE = -6
U = 2.0 ** -24
ACC_BOUND_REL = 2.0 ** -12            # the accumulation allowance of eps_rel in certify_kernel


def _native():
    from kaito_b200 import _native
    return _native


PASS_NAMES = {0: "TF32", 1: "BF16_SPLIT", 2: "BF16_SHADOW", 3: "BF16_HOST"}
RATIOS = {}                           # (pass, dpad) -> largest observed error / bound


def hi_split(x):
    """the high halves of split rows as fp32 values"""
    return (split_hi(np.ascontiguousarray(x, np.float32).view(np.uint32)) << 16).astype(np.uint32).view(np.float32)


def operands(x, q, tc_pass, split):
    if tc_pass == 0:
        return tf32_trunc(x), tf32_trunc(q)
    if tc_pass == 1:
        return hi_split(x), bf16_rn(q)
    return bf16_rn(x), bf16_rn(q)


def k_steps(dpad, tc_pass):
    return dpad // (8 if tc_pass == 0 else 16)


def dump_xn(ix, q, tc_pass, n):
    """(a [NQ, S], xn [n]): xn from a padded column, from a one-query dump when the batch fills its bucket"""
    a = ix.debug_tc_dump_pass(q, tc_pass)
    nq, NQ, S = len(q), a.shape[0], a.shape[1]
    assert NQ == (64 if nq <= 64 else 128 if nq <= 128 else 256) and S == -(-n // 128) * 128
    assert np.isposinf(a[:, n:]).all(), "rows past the end must dump +inf"
    if nq < NQ:
        xn = a[nq, :n]
        assert np.array_equal(a[nq:, :n], np.broadcast_to(xn, (NQ - nq, n))), "zero queries must return |x|^2"
    else:
        xn = ix.debug_tc_dump_pass(q[:1], tc_pass)[1, :n]
    return a, xn


def check_pass(ix, x, q, tc_pass, exact=False, what=""):
    """the dump of one pass against fp64 over its operands; returns (acc rebuilt [nq, n], reference [nq, n], bound)"""
    n, dpad = x.shape
    split = ix.stats().dim_padded % 64 == 0 and tc_pass != 3
    a, xn = dump_xn(ix, q, tc_pass, n)
    nq = len(q)
    x64 = x.astype(np.float64)
    # the stored |x|^2 itself: row_norms_kernel, at most dpad / 128 + 9 roundings per term
    xn_ref = (x64 ** 2).sum(1)
    assert (np.abs(xn - xn_ref) <= (dpad // 128 + 9) * U * xn_ref * 1.0001 + 1e-37).all(), f"{what}: |x|^2"
    xo, qo = operands(x, q, tc_pass, split)
    ref = qo.astype(np.float64) @ xo.astype(np.float64).T
    absref = np.abs(qo.astype(np.float64)) @ np.abs(xo.astype(np.float64)).T
    a64 = a[:nq, :n].astype(np.float64)
    acc = (xn.astype(np.float64)[None, :] - a64) / 2.0
    err = np.abs(acc - ref)
    if exact:                           # integer data: every operand, product and partial sum is exact
        assert np.array_equal(a[:nq, :n].astype(np.float64), xn_ref[None, :] - 2.0 * ref), f"{what}: not exact"
        return acc, ref, np.zeros_like(ref)
    bound = k_steps(dpad, tc_pass) * 2.0 ** -23 * absref + 2.0 ** -25 * np.abs(a64) + 1e-30
    ratio = float((err / bound).max())
    key = (PASS_NAMES[tc_pass], dpad)
    RATIOS[key] = max(RATIOS.get(key, 0.0), ratio)
    print(f"{what} {PASS_NAMES[tc_pass]} dpad={dpad} n={n} nq={nq}: max err / bound = {ratio:.3g}")
    if ratio > 1.0:
        j, r = np.unravel_index(np.argmax(err / bound), err.shape)
        raise AssertionError(f"{what} {PASS_NAMES[tc_pass]}: query {j} row {r}: acc {acc[j, r]!r} ref {ref[j, r]!r} "
                             f"err {err[j, r]:.3g} bound {bound[j, r]:.3g}")
    return acc, ref, bound


# ------------------------------------------------------------------------------------------------------------- data
def crafted_rows(n, dpad, seed):
    """fp32 values whose low halves sit at the rounding edges: ties (lo == 0x8000, odd and even high halves), just below
    and above the midpoint, mantissas that carry into the exponent, mixed signs; exponents 2^-4 .. 2^3"""
    g = np.random.default_rng(seed)
    sign = g.integers(0, 2, (n, dpad), dtype=np.uint32) << 31
    expo = g.integers(123, 131, (n, dpad), dtype=np.uint32) << 23
    mant = g.integers(0, 128, (n, dpad), dtype=np.uint32) << 16
    kind = g.integers(0, 5, (n, dpad))
    lo = np.choose(kind, [np.full((n, dpad), 0x8000, np.uint32), np.full((n, dpad), 0x7FFF, np.uint32),
                          np.full((n, dpad), 0x8001, np.uint32), g.integers(0, 1 << 16, (n, dpad), dtype=np.uint32),
                          np.full((n, dpad), 0xFFFF, np.uint32)]).astype(np.uint32)
    mant = np.where(kind == 4, np.uint32(0x7F << 16), mant)       # 0x..7FFFFF: rounding up carries into the exponent
    return (sign | expo | mant | lo).view(np.float32)


def tie_rows(n, dpad, seed):
    """every element a positive exact tie (lo == 0x8000) on an odd high half in [1, 2): round-to-even rounds every one up
    by 2^-7, the split rows' high halves keep every one down, so the two products differ by 2^-7 sum q"""
    g = np.random.default_rng(seed)
    hi = np.uint32(0x3F80) + 2 * g.integers(0, 64, (n, dpad), dtype=np.uint32) + 1
    return ((hi << 16) | 0x8000).astype(np.uint32).view(np.float32)


def integer_rows(n, dpad, seed, lim=8):
    return np.random.default_rng(seed).integers(-lim, lim + 1, (n, dpad)).astype(np.float32)


# --------------------------------------------------------------------------------------------------------- contexts
@pytest.fixture(scope="module")
def ctx_bf16():
    """split rows with a bf16 shadow: one index serves the TF32 (TC_TF32S), BF16_SPLIT and BF16_SHADOW passes"""
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


def _index(ctx, name, x):
    ix = ctx.create_index(name, x.shape[1])
    ix.add(np.arange(len(x), dtype=np.uint64), x)
    return ix


# ----------------------------------------------------------------------------------- values at every shape and bucket
# (dpad, n, nq): every NQ bucket and its padding edge, every tile-tail shape (n % 128 = 1, 127, 0, and longer tails)
SHAPES = [(64, 1, 1), (64, 127, 63), (64, 129, 64), (128, 128, 65), (128, 3000, 129), (384, 1000, 256), (768, 2049, 128),
          (768, 129, 1), (1024, 2000, 65), (4096, 1500, 63), (16384, 1024, 64), (16384, 129, 256)]


@pytest.mark.parametrize("dpad,n,nq", SHAPES)
def test_passes_match_fp64_on_synth_data(ctx_bf16, oracle, dpad, n, nq):
    N = _native()
    x = oracle.synth_dense(n, dpad, seed=dpad + n)
    q = oracle.synth_queries(x, nq, seed=nq + 7)
    ix = _index(ctx_bf16, f"syn_{dpad}_{n}_{nq}", x)
    try:
        for p in (N.TC_PASS_BF16_SPLIT, N.TC_PASS_BF16_SHADOW, N.TC_PASS_TF32):
            check_pass(ix, x, q, p, what="synth")
    finally:
        ix.drop()


@pytest.mark.parametrize("dim,n,nq", [(96, 129, 65), (800, 1000, 129), (800, 1, 256)])
def test_tf32_pass_on_plain_rows(ctx_bf16, oracle, dim, n, nq):
    """dpad % 64 == 32 keeps plain fp32 rows: TC_TF32, and no bf16 pass (the shadow is not used at this width)"""
    N = _native()
    x = oracle.synth_dense(n, dim, seed=dim)
    q = oracle.synth_queries(x, nq, seed=3)
    ix = _index(ctx_bf16, f"plain_{dim}_{n}", x)
    try:
        check_pass(ix, x, q, N.TC_PASS_TF32, what="plain")
        with pytest.raises(N.KragError):
            ix.debug_tc_dump_pass(q, N.TC_PASS_BF16_SPLIT)
    finally:
        ix.drop()


@pytest.mark.parametrize("dpad,n,nq", [(64, 129, 65), (1024, 700, 63), (16384, 130, 2)])
def test_passes_on_crafted_rounding_edges(ctx_bf16, dpad, n, nq):
    N = _native()
    x = crafted_rows(n, dpad, seed=dpad)
    q = crafted_rows(nq, dpad, seed=dpad + 1)
    ix = _index(ctx_bf16, f"edge_{dpad}", x)
    try:
        for p in (N.TC_PASS_BF16_SPLIT, N.TC_PASS_BF16_SHADOW, N.TC_PASS_TF32):
            check_pass(ix, x, q, p, what="crafted")
    finally:
        ix.drop()


@pytest.mark.parametrize("dpad,n,nq", [(128, 300, 64), (768, 129, 65), (16384, 200, 129)])
def test_passes_exact_on_integer_data(ctx_bf16, dpad, n, nq):
    """small integers are exact in bf16 and TF32 and so is every partial sum: the dump must equal fp64 bit for bit"""
    N = _native()
    x = integer_rows(n, dpad, seed=dpad)
    q = integer_rows(nq, dpad, seed=dpad + 5)
    ix = _index(ctx_bf16, f"int_{dpad}", x)
    try:
        for p in (N.TC_PASS_BF16_SPLIT, N.TC_PASS_BF16_SHADOW, N.TC_PASS_TF32):
            check_pass(ix, x, q, p, exact=True, what="integer")
    finally:
        ix.drop()


def test_split_pass_rounds_ties_toward_zero(ctx_bf16):
    """on rows of exact ties the split pass's operand is the high half rounded toward zero: a reference that rounds the
    row to nearest even (the shadow's operand) must fail the bound, and the shadow pass must fail the split reference"""
    N = _native()
    n, dpad, nq = 130, 128, 3
    x = tie_rows(n, dpad, seed=1)
    q = np.abs(integer_rows(nq, dpad, seed=2)) + 1.0           # positive: the per-element differences add up
    ix = _index(ctx_bf16, "ties", x)
    try:
        acc_s, ref_s, bound_s = check_pass(ix, x, q, N.TC_PASS_BF16_SPLIT, what="ties")
        acc_h, ref_h, bound_h = check_pass(ix, x, q, N.TC_PASS_BF16_SHADOW, what="ties")
        assert (np.abs(acc_s - ref_h) > bound_s).all(), "the split pass matched a round-to-even reference"
        assert (np.abs(acc_h - ref_s) > bound_h).all(), "the shadow pass matched the ties-toward-zero reference"
    finally:
        ix.drop()


# --------------------------------------------------------------------------------------------- the error allowances
@pytest.mark.parametrize("tc_pass,eps_rel", [(1, EPS_BF16), (2, EPS_BF16), (0, EPS_TF32)])
def test_eps_rel_holds_on_positive_data_at_dpad_16384(ctx_bf16, tc_pass, eps_rel):
    """all-positive rows and queries at the widest rows (1,024 bf16 / 2,048 tf32 K steps): no cancellation, so the
    accumulation error is as large relative to |x||q| as it gets.  Against the true fp32 inputs the accumulation part
    must stay within 2^-12 |x||q| and the whole error within eps_rel |x||q|."""
    n, dpad, nq = 257, 16384, 5
    g = np.random.default_rng(16)
    x = g.random((n, dpad), dtype=np.float32) + np.float32(2.0 ** -20)
    q = g.random((nq, dpad), dtype=np.float32) + np.float32(2.0 ** -20)
    ix = _index(ctx_bf16, f"pos_{tc_pass}", x)
    try:
        acc, ref, _ = check_pass(ix, x, q, tc_pass, what="positive")
        norms = np.linalg.norm(q.astype(np.float64), axis=1)[:, None] * np.linalg.norm(x.astype(np.float64), axis=1)[None, :]
        acc_rel = np.abs(acc - ref) / norms
        whole_rel = np.abs(acc - q.astype(np.float64) @ x.astype(np.float64).T) / norms
        print(f"{PASS_NAMES[tc_pass]} dpad=16384 positive: accumulation {acc_rel.max():.3g} |x||q| "
              f"(2^-12 = {ACC_BOUND_REL:.3g}), whole {whole_rel.max():.3g} |x||q| (eps_rel = {eps_rel:.3g})")
        assert acc_rel.max() <= ACC_BOUND_REL and whole_rel.max() <= eps_rel
    finally:
        ix.drop()


def test_bf16_error_on_the_certificate_construction(oracle):
    """the adversarial corpus of test_tc_certificate_bound.py: the bf16 passes' measured error on its target row exceeds
    2^-8 + 2^-12 (a halved eps_rel would not cover it) and stays within eps_rel, and the search, whose certificate must
    refuse that query, still returns the oracle's answer"""
    from tests import test_tc_certificate_bound as adv
    N = _native()
    x, q_adv, _ = adv.adversarial_corpus(1)
    q = np.concatenate([q_adv[None, :], oracle.synth_queries(x, 15, seed=41)])
    c = N.Context(device_id=0, dense_mode=N.DENSE_TC_BF16)    # its own: the search below switches the context's mode
    ix = _index(c, "adv", x)
    try:
        xs, qa = x[adv.TARGET_ROW].astype(np.float64), q_adv.astype(np.float64)
        norm = np.linalg.norm(xs) * np.linalg.norm(qa)
        xn = float(np.float32((xs ** 2).sum()))
        for p in (N.TC_PASS_BF16_SPLIT, N.TC_PASS_BF16_SHADOW):
            a = ix.debug_tc_dump_pass(q[:1], p)
            acc = (float(a[1, adv.TARGET_ROW]) - float(a[0, adv.TARGET_ROW])) / 2.0   # padded column: xn
            assert a[1, adv.TARGET_ROW] == np.float32(xn)
            rel = abs(acc - xs @ qa) / norm
            print(f"{PASS_NAMES[p]}: error on the target row {rel:.6g} |x||q|")
            assert 2.0 ** -8 + 2.0 ** -12 < rel <= EPS_BF16
        ix.set_dense_mode(N.DENSE_TC)
        fb0 = N.load().krag_tc_fallback_queries()
        dist, ordn = ix.search_dense(q, 1)
        fb = N.load().krag_tc_fallback_queries() - fb0
        rd, ro = oracle.dense_topk(x, q, 1)
        assert np.array_equal(ordn, ro) and np.array_equal(dist, rd)
        assert fb >= 1 and ro[0, 0] == adv.TARGET_ROW
        assert N.last_dense_kernel()[1] in (1, 5)
    finally:
        ix.drop()
        c.close()


# ------------------------------------------------------------------------------------------------- shadow freshness
def _fresh(ix, what, tc_pass=2, nq=33, seed=0):
    """the shadow (or host copy) pass against the reference built from the rows as read back"""
    n = int(ix.stats().n_rows)
    x = ix.read_rows(0, n)
    q = integer_rows(nq, x.shape[1], seed=seed + 99)
    exact = bool(np.array_equal(x, np.round(x)) and np.abs(x).max() <= 16)
    check_pass(ix, x, q, tc_pass, exact=exact, what=what)


def test_shadow_follows_adds_fill_mode_switch_compact_and_load(oracle, tmp_path):
    N = _native()
    dpad = 128
    x = integer_rows(1500, dpad, seed=11)
    c = N.Context(device_id=0, dense_mode=N.DENSE_TC_BF16)
    d = N.Context(device_id=0)
    try:
        ix = c.create_index("fresh_add", dpad)
        for a, b in ((0, 100), (100, 641), (641, 1500)):        # adds in several batches
            ix.add(np.arange(a, b, dtype=np.uint64), x[a:b])
            _fresh(ix, f"add[{a}:{b}]")
        ix.remove(np.arange(0, 1500, 3, dtype=np.uint64))       # remove + compact: every later row moves
        ix.compact()
        assert ix.stats().n_rows == 1000
        _fresh(ix, "compact")
        path = str(tmp_path / "fresh.krag")
        ix.persist(path)
        ix.drop()
        ld = c.load_index("fresh_load", path)
        _fresh(ld, "persist/load")
        ld.drop()

        sf = c.create_index("fresh_fill", 768)                  # synth_fill writes rows, norms and shadow on the device
        sf.synth_fill(1000, row_base=5, seed=3, vocab=0)
        _fresh(sf, "synth_fill", nq=65)
        sf.drop()

        sw = d.create_index("fresh_switch", dpad)               # split rows without a shadow, then TC_BF16 builds it
        sw.add(np.arange(700, dtype=np.uint64), x[:700])
        with pytest.raises(N.KragError) as e:
            sw.debug_tc_dump_pass(x[:1], N.TC_PASS_BF16_SHADOW)
        assert e.value.code == KRAG_E_STATE
        sw.set_dense_mode(N.DENSE_TC_BF16)
        _fresh(sw, "set_dense_mode")
        sw.add(np.arange(700, 1500, dtype=np.uint64), x[700:])  # appends convert into the shadow built from split rows
        _fresh(sw, "add after set_dense_mode")
        sw.drop()
    finally:
        c.close()
        d.close()


def test_shadow_follows_a_two_shard_redeal(oracle, monkeypatch):
    """round-robin shards compacted together (krag_redeal_*): rows move between the shards, and each shard's shadow with them"""
    from tests.test_gpu_sharded_compact import LoopbackA2A, RR
    from kaito_b200 import sharded
    monkeypatch.setattr(sharded, "dist", LoopbackA2A)
    monkeypatch.setenv("KRAG_P2P", "0")
    N = _native()
    n, dpad, vocab = 3001, 64, 300
    x = integer_rows(n, dpad, seed=21)
    csr = oracle.synth_sparse(n, vocab, 22, mean_len=8.0)
    c = N.Context(device_id=0, dense_mode=N.DENSE_TC_BF16)
    sh = RR(sharded, c, "redeal", x, csr, vocab, 2)
    try:
        sh.commit()
        dead = np.random.default_rng(23).random(n) < 0.3
        sh.remove(np.flatnonzero(dead))
        sh.commit()
        sh.compact(window_rows=500)
        live = np.flatnonzero(~dead)
        for s, ix in enumerate(sh.ix):
            assert np.array_equal(ix.read_rows(0, int(ix.stats().n_rows)), x[live[s::2]])
            _fresh(ix, f"redeal shard {s}")
    finally:
        sh.drop()
        c.close()


def test_host_copy_follows_compact(ctx_host):
    N = _native()
    dpad = 192
    x = integer_rows(2000, dpad, seed=31)
    ix = _index(ctx_host, "host_compact", x)
    try:
        _fresh(ix, "host add", tc_pass=N.TC_PASS_BF16_HOST)
        for p in (N.TC_PASS_TF32, N.TC_PASS_BF16_SPLIT, N.TC_PASS_BF16_SHADOW):
            with pytest.raises(N.KragError):
                ix.debug_tc_dump_pass(x[:1], p)
        ix.remove(np.arange(0, 2000, 5, dtype=np.uint64))
        ix.compact()
        _fresh(ix, "host compact", tc_pass=N.TC_PASS_BF16_HOST)
    finally:
        ix.drop()


# ---------------------------------------------------------------------------------------------- candidate emission
def _emission(ix, x, q, alive, tc_pass, thr_pad, what, exact=False):
    """krag_debug_tc_prune against the dump: thr per real query at the ~5 % quantile of its alive rows; thr_pad for the
    padded columns (whose zero queries give a = xn).  Returns (counts, expected sets) for further checks."""
    n = len(x)
    a, xn = dump_xn(ix, q, tc_pass, n)
    nq, NQ = len(q), a.shape[0]
    a = a[:, :n].astype(np.float64)
    thr = np.empty(NQ, np.float32)
    for j in range(nq):
        thr[j] = np.quantile(a[j, alive], 0.05)
    thr[nq:] = thr_pad(NQ - nq, xn)
    cap = n
    counts, rows = ix.debug_tc_prune(q, thr, cap, tc_pass)
    expect = []
    for j in range(NQ):
        t = float(thr[j])
        e = np.flatnonzero((a[j] < t) & alive)
        got = rows[j, :min(int(counts[j]), cap)]
        assert int(counts[j]) == len(got) <= cap, f"{what}: query {j} count {counts[j]}"
        assert len(np.unique(got)) == len(got) and (got < n).all() and alive[got].all(), f"{what}: query {j} bad rows"
        if exact:
            band = np.zeros(n, bool)
        else:   # |a - thr| within the epilogue's and the dump's roundings: 2^-23 (|a| + |2 acc| + |thr|) covers both
            band = np.abs(a[j] - t) <= 2.0 ** -23 * (np.abs(a[j]) + np.abs(xn - a[j]) + abs(t))
        gs, es = set(got.tolist()), set(e.tolist())
        diff = gs.symmetric_difference(es)
        assert all(band[r] for r in diff), f"{what}: query {j}: rows {sorted(diff)[:8]} differ outside the rounding band"
        expect.append(es)
    return thr, counts, rows


@pytest.mark.parametrize("tc_pass", [0, 1, 2])
def test_candidate_emission_with_tombstones_tail_and_padding(ctx_bf16, oracle, tc_pass):
    """n = 1000 (a 104-row tail tile), 65 queries (63 padded columns in the 128 bucket), 10 % tombstones.  Padded columns
    get thresholds that admit everything, half the rows, or nothing: their lists must be exactly that, and the real
    queries' lists must not change with them"""
    n, dpad, nq = 1000, 256, 65
    x = oracle.synth_dense(n, dpad, seed=51)
    q = oracle.synth_queries(x, nq, seed=52)
    ix = _index(ctx_bf16, f"emit_{tc_pass}", x)
    try:
        dead = np.random.default_rng(53).choice(n, 100, replace=False)
        ix.remove(dead.astype(np.uint64))
        alive = np.ones(n, bool)
        alive[dead] = False

        def wide(k, xn):
            t = np.full(k, np.inf, np.float32)
            t[1::3] = np.float32(np.median(xn))
            t[2::3] = -np.inf
            return t

        thr, counts, full = _emission(ix, x, q, alive, tc_pass, wide, f"{PASS_NAMES[tc_pass]} emission")
        assert counts[nq] == alive.sum()                          # +inf: every alive row, none past n, no tombstone
        assert counts[nq + 2] == 0
        # the padded columns as the search runs them (-inf: nothing) leave the real queries' lists as they were
        thr_q = np.concatenate([thr[:nq], np.full(len(thr) - nq, -np.inf, np.float32)])
        counts_q, rows_q = ix.debug_tc_prune(q, thr_q, n, tc_pass)
        assert np.array_equal(counts_q[:nq], counts[:nq]) and (counts_q[nq:] == 0).all()
        for j in range(nq):
            assert set(rows_q[j, :counts_q[j]].tolist()) == set(full[j, :counts[j]].tolist()), f"query {j}"
        # cap overflow: the count goes on, the stored rows are a subset of the full list
        cap = 8
        counts_c, rows_c = ix.debug_tc_prune(q, thr, cap, tc_pass)
        assert np.array_equal(counts_c, counts)
        for j in range(nq):
            assert counts[j] > cap
            assert set(rows_c[j].tolist()) <= set(full[j, :counts[j]].tolist())
    finally:
        ix.drop()


@pytest.mark.parametrize("tc_pass", [0, 1, 2])
def test_candidate_test_is_strict_on_integer_data(ctx_bf16, tc_pass):
    """exact arithmetic: thr set to some rows' own a; those rows are not candidates (a < thr), the rows just below are"""
    n, dpad, nq = 777, 128, 7
    x = integer_rows(n, dpad, seed=61)
    q = integer_rows(nq, dpad, seed=62)
    ix = _index(ctx_bf16, f"strict_{tc_pass}", x)
    try:
        a = ix.debug_tc_dump_pass(q, tc_pass)[:, :n].astype(np.float64)
        alive = np.ones(n, bool)
        NQ = 64
        thr = np.full(NQ, -np.inf, np.float32)
        for j in range(nq):
            thr[j] = np.sort(a[j])[n // 10]                       # some row's exact a
        counts, rows = ix.debug_tc_prune(q, thr, n, tc_pass)
        for j in range(nq):
            got = set(rows[j, :counts[j]].tolist())
            assert got == set(np.flatnonzero(a[j] < thr[j]).tolist()), f"query {j}"
            at = np.flatnonzero(a[j] == thr[j])
            assert len(at) >= 1 and not (set(at.tolist()) & got), f"query {j}: a row with a == thr was emitted"
        _emission(ix, x, q, alive, tc_pass, lambda k, xn: np.full(k, -np.inf, np.float32), "integer emission", exact=True)
    finally:
        ix.drop()


def test_candidate_emission_host_copy(ctx_host, oracle):
    N = _native()
    n, dpad, nq = 900, 128, 3
    x = oracle.synth_dense(n, dpad, seed=71)
    q = oracle.synth_queries(x, nq, seed=72)
    ix = _index(ctx_host, "emit_host", x)
    try:
        dead = np.arange(0, n, 7)
        ix.remove(dead.astype(np.uint64))
        alive = np.ones(n, bool)
        alive[dead] = False
        check_pass(ix, x, q, N.TC_PASS_BF16_HOST, what="host")
        _emission(ix, x, q, alive, N.TC_PASS_BF16_HOST, lambda k, xn: np.full(k, np.inf, np.float32), "host emission")
    finally:
        ix.drop()


def test_report_ratios():
    """the largest observed error over the derived bound per pass and dpad (printed with -s; every value is <= 1)"""
    for key in sorted(RATIOS):
        print(f"max err / bound {key[0]:12s} dpad {key[1]:6d}: {RATIOS[key]:.4f}")
    assert all(v <= 1.0 for v in RATIOS.values())
