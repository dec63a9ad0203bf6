"""CPU check of the slack term of K2's exactness certificate (certify_kernel, certify_slack_rel in dense_tc.cu).

The certificate passes a query when  D_P <= thr + |q|^2 - 2 eps - slack.  eps covers the main pass's dot product; the
slack covers every other fp32 rounding between the pruned row's true distance and the D_P it is compared with:
  |x|^2   row_norms_kernel: per lane, each float4 is summed as ((x0^2 + x1^2) + x2^2) + x3^2 (a square and 3 adds) and
          added to the lane's running sum (dpad / 128 float4s per lane), then a 5-step butterfly:  mx = dpad / 128 + 9
  |q|^2   certify_kernel: per lane an FFMA chain over dpad / 32 elements, then the butterfly:  mq = dpad / 32 + 5
  D1      K1's fp32 distance of the pruned row (fetch_rule_constants):  mk = dpad / 32 + 7, with D <= 2 (|x|^2 + |q|^2)
  and the epilogue's add plus the certificate's three adds: 9 roundings of operands below 3 (|x|^2max + |q|^2).
A sum whose terms pass through at most m roundings to nearest is within gamma_m = m u / (1 - m u) of its exact value
(u = 2^-24, Higham Lemma 3.1), so the slack must be at least
    gamma_mx |x|^2max + gamma_mq |q|^2 + 2 gamma_mk (|x|^2max + |q|^2) + 9 u (...)
The constant 4e-6 (1 + |q|^2 + |x|^2max) the certificate used before covers that only up to dpad 416; K2 accepts rows
up to dpad 16384, where the worst case for unit vectors is about 14 times larger.  The slack is now derived from dpad.
"""
import numpy as np

U = 2.0 ** -24
LANES = 32
OLD_SLACK = 4e-6


def gamma(m):
    return m * U / (1.0 - m * U)


def roundings(dpad):
    """(mx, mq, mk): roundings per term of |x|^2, |q|^2 and K1's distance"""
    return dpad // 128 + 9, dpad // LANES + 5, dpad // LANES + 7


def required(dpad, xmax, qn):
    """worst-case fp32 error outside the main pass's dot product, for given |x|^2max and |q|^2"""
    mx, mq, mk = roundings(dpad)
    return gamma(mx) * xmax + gamma(mq) * qn + 2.0 * gamma(mk) * (xmax + qn) + gamma(9) * (xmax + qn)


def slack_rel(dpad):
    """certify_slack_rel (dense_tc.cu), restated"""
    mx, mq, mk = roundings(dpad)
    m = max(mx, mq) + 2.0 * mk + 9.0
    c = m * U / (1.0 - m * U)
    return float(np.nextafter(np.float32(c), np.float32(np.inf))) if c > OLD_SLACK else float(np.float32(OLD_SLACK))


DPADS = range(32, 16384 + 1, 32)     # every padded dimension the index accepts
NORMS = [(1.0, 1.0), (1.0, 1e-3), (1e-3, 1.0), (1e4, 1e4), (1e6, 1.0), (1.0, 1e6)]


def test_derived_slack_covers_the_worst_case_at_every_dpad():
    for dpad in DPADS:
        s = slack_rel(dpad)
        for xmax, qn in NORMS:
            assert required(dpad, xmax, qn) <= s * (1.0 + qn + xmax), (dpad, xmax, qn)


def test_old_constant_falls_short_for_wide_rows():
    short = [d for d in DPADS if any(required(d, xm, qn) > OLD_SLACK * (1.0 + qn + xm) for xm, qn in NORMS)]
    assert short and min(short) == 448 and short == [d for d in DPADS if d >= 448]
    assert required(16384, 1.0, 1.0) / (OLD_SLACK * 3.0) > 13.0      # ~14x at the widest rows


def test_slack_is_unchanged_where_the_old_constant_sufficed():
    """narrow rows keep 4e-6 exactly: the change only adds fallbacks where the old slack was unsound"""
    for dpad in DPADS:
        if dpad < 448:
            assert slack_rel(dpad) == float(np.float32(OLD_SLACK)), dpad
        else:
            assert slack_rel(dpad) > OLD_SLACK
    assert 5.9e-6 < slack_rel(768) < 6.0e-6 and 9.3e-5 < slack_rel(16384) < 9.4e-5


def test_slack_stays_far_below_the_dot_product_allowance():
    """even at dpad 16384 the slack is < 2 % of 2 eps for unit vectors (eps_rel >= 2^-9 + 2^-12): the certificate's
    margin, and so its fallback rate on real data, is set by eps, not by the slack"""
    eps_tf32 = 2.0 ** -9 + 2.0 ** -12
    for dpad in DPADS:
        assert slack_rel(dpad) * 3.0 < 0.1 * 2.0 * eps_tf32
