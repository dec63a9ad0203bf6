"""GPU tests of the fp16 precision mode of K5 (krag_embedder_set_precision(KRAG_PRECISION_FP16)): fp16 operands, one
tensor-core product per step, fp32 accumulation / residual stream / LayerNorm / softmax / head.

The single-plane GEMM is exact on fp16 inputs up to fp32 accumulation, so it is held to the split GEMM's bound.  The forward is
held to two rules: its logit (embedding) error against fp64 is at most that of torch under bf16 autocast on the same inputs and
the same GPU, and the sigmoid score moves by at most SCORE_TOL_FP16.  The default mode must not notice any of it: its outputs
are compared bit for bit around a switch to fp16 and back."""
import copy

import numpy as np
import pytest

from tests import bert_reference as br
from tests.test_gpu_rerank import CE_MODELS, _all_scores, _encoder, _pairs_of, _random_pairs, _state

# Twice the worst sigmoid-score error measured over the cases below: 6.1e-4 at hidden 1024, 4.8e-4 at the CE_MODELS shapes
# (MiniLM-L6 stressed); torch bf16 autocast on the same pairs: 5.4e-3 and 8.9e-3 (H100 80GB HBM3, 700 W power limit)
SCORE_TOL_FP16 = 1.2e-3
# the first 17 shapes of test_gpu_embed.test_gemm_tf32_matches_numpy: M edges 1, 127+, 129, ragged; K = 64 ... 4096
GEMM_SHAPES = [(10, 128, 64, False, False), (300, 384, 384, False, True), (1000, 1152, 384, False, False),
               (257, 1536, 384, True, False), (129, 384, 1536, False, True), (4096, 768, 768, True, True),
               (1, 768, 768, False, False), (16, 2304, 768, False, False), (16, 3072, 768, True, False),
               (100, 768, 3072, False, True), (128, 384, 384, False, True), (7, 1024, 4096, False, True),
               (512, 768, 768, False, True), (400, 768, 3072, False, True), (512, 2304, 768, False, False),
               (1024, 768, 3072, False, True), (600, 1024, 4096, False, False)]


def _gelu(x):
    from scipy.special import erf
    return 0.5 * x * (1 + erf(x / np.sqrt(2)))


def _h(x):
    """x rounded to fp16 (round to nearest even), as fp32"""
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def _gemm_ref(A, B, bias, R, gelu):
    ref = A.astype(np.float64) @ B.astype(np.float64).T + bias
    if gelu:
        ref = _gelu(ref)
    return ref + R if R is not None else ref


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,gelu,res", GEMM_SHAPES)
def test_gemm_f16_is_exact_on_fp16_inputs(ctx, M, N, K, gelu, res):
    from kaito_b200 import _native
    g = np.random.default_rng(M + N + K)
    A = _h(g.standard_normal((M, K)))
    B = _h(g.standard_normal((N, K)) / np.sqrt(K))
    bias = g.standard_normal(N).astype(np.float32)
    R = g.standard_normal((M, N)).astype(np.float32) if res else None
    ref = _gemm_ref(A, B, bias, R, gelu)
    for tile_n in (0, 32, 64, 128, 256):         # 0: the forward's own plan (split-K for a handful of rows)
        if N % 256 and tile_n == 256:
            continue
        err = np.abs(_native.debug_gemm_f16(ctx, A, B, bias, R, gelu, tile_n) - ref)
        print(f"gemm f16 {M}x{N}x{K} tile {tile_n}: max {err.max():.2e} mean {err.mean():.2e}")
        # products of fp16 numbers are exact in fp32: what is left is fp32 accumulation, the split GEMM's bound
        assert err.max() < 5e-5 and err.mean() < 5e-6, (tile_n, err.max(), err.mean())
    # fp32 inputs: the product of the fp16-rounded inputs
    A32 = g.standard_normal((M, K)).astype(np.float32)
    B32 = (g.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    err = np.abs(_native.debug_gemm_f16(ctx, A32, B32, bias, R, gelu) - _gemm_ref(_h(A32), _h(B32), bias, R, gelu))
    assert err.max() < 5e-5 and err.mean() < 5e-6, (err.max(), err.mean())


@pytest.mark.gpu
def test_gemm_f16_saturates_and_refuses_bad_tiles(ctx):
    from kaito_b200 import _native
    A = np.zeros((4, 64), np.float32); A[:, 0] = 1e6                       # past fp16's range: rounds to 65504, not inf
    B = np.zeros((128, 64), np.float32); B[:, 0] = 1.0
    got = _native.debug_gemm_f16(ctx, A, B, np.zeros(128, np.float32))
    assert np.array_equal(got, np.full((4, 128), 65504.0, np.float32))
    with pytest.raises(_native.KragError):
        _native.debug_gemm_f16(ctx, A, B, np.zeros(128, np.float32), tile_n=256)      # N % 256 != 0
    with pytest.raises(_native.KragError):
        _native.debug_gemm_tf32(ctx, A, np.zeros((256, 64), np.float32), np.zeros(256, np.float32), tile_n=256)


# ------------------------------------------------------------------------------------------------ torch bf16 yardstick
def _bf16_logits(ref, pairs):
    """logits of torch's BertForSequenceClassification under bf16 autocast on the GPU, each pair alone"""
    import torch
    m = copy.deepcopy(ref.m32).cuda()
    out = []
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for ids, seg in pairs:
            tt = (np.arange(len(ids)) >= seg).astype(np.int64)
            out.append(float(m(input_ids=torch.tensor(np.asarray(ids, np.int64)[None]).cuda(),
                               token_type_ids=torch.tensor(tt[None]).cuda()).logits[0, 0].float()))
    return np.asarray(out, np.float64)


def _bf16_pools(ref, toks):
    """(CLS rows, token means), L2-normalised, of torch's BertModel under bf16 autocast on the GPU"""
    import torch
    m = copy.deepcopy(ref.m64).float().cuda()
    cls, mean = [], []
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for t in toks:
            h = m(input_ids=torch.tensor(np.asarray(t, np.int64)[None]).cuda()).last_hidden_state[0].float().cpu().numpy().astype(np.float64)
            cls.append(h[0] / np.linalg.norm(h[0])); mean.append(h.mean(0) / np.linalg.norm(h.mean(0)))
    return np.stack(cls), np.stack(mean)


def _check_logits(label, cfg, state, enc, flat, toff, seg, poff, idx):
    """fp16-mode logits and sigmoid scores of pairs `idx` against fp64, next to torch bf16 autocast's"""
    from kaito_b200 import _native
    enc.set_precision("fp16")
    logit = _all_scores(enc, flat, toff, seg, poff, _native.RERANK_IDENTITY)
    score = _all_scores(enc, flat, toff, seg, poff, _native.RERANK_SIGMOID)
    ref = br.Fp64CrossEncoder(cfg, state)
    pairs = _pairs_of(flat, toff, seg, idx)
    l64 = ref.logits(pairs)[0]
    b16 = _bf16_logits(ref, pairs)
    k5, t16 = float(np.abs(logit[idx] - l64).max()), float(np.abs(b16 - l64).max())
    ds = float(np.abs(score[idx] - 1.0 / (1.0 + np.exp(-l64))).max())
    ds16 = float(np.abs(1.0 / (1.0 + np.exp(-b16)) - 1.0 / (1.0 + np.exp(-l64))).max())
    print(f"rerank fp16 vs fp64 | {label} | {len(idx)} of {len(toff) - 1} pairs, {int(toff[-1])} tok | logit err {k5:.2e} | "
          f"torch bf16 {t16:.2e} | ratio {k5 / t16:.3f} | sigmoid err {ds:.2e} | torch bf16 sigmoid err {ds16:.2e}")
    assert k5 <= t16, (label, k5, t16)
    assert ds <= SCORE_TOL_FP16, (label, ds)
    return logit, score


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["bench", "stressed"])
@pytest.mark.parametrize("model", list(CE_MODELS))
def test_fp16_logits_match_fp64_within_torch_bf16(ctx, model, regime):
    if model == "base" and regime == "stressed":
        pytest.skip("the stressed regime runs at the MiniLM and TinyBERT shapes")
    cfg = CE_MODELS[model]
    state = _state(cfg, regime)
    enc = _encoder(ctx, cfg, state)
    g = np.random.default_rng(5)
    # the pair mix of test_gpu_rerank.test_logits_match_fp64: 512-token pairs, an empty query, empty passages
    flat, toff, seg, poff = _random_pairs(g, 8, 30, long_every=37)
    edge = _random_pairs(g, 2, 3, q_len=(0, 0), d_len=(0, 1))
    flat = np.concatenate([flat, edge[0]]); toff = np.concatenate([toff, toff[-1] + edge[1][1:]])
    seg = np.concatenate([seg, edge[2]]); poff = np.concatenate([poff, poff[-1] + edge[3][1:]])
    lens = np.diff(toff)
    n = len(lens)
    idx = sorted(set(br.sample(lens.tolist(), 12 if model == "base" else 20).tolist()) | {n - 1, n - 2, n - 6}
                 | set(np.flatnonzero(lens == 512)[:2].tolist()))
    _check_logits(f"{model} {regime}", cfg, state, enc, flat, toff, seg, poff, idx)
    enc.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("label,cfg,long_len", [
    ("head dim 32", dict(num_hidden_layers=2, hidden_size=256, num_attention_heads=8, intermediate_size=1024, vocab_size=30522,
                         max_position_embeddings=512), 0),
    ("hidden 1024", dict(num_hidden_layers=2, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, vocab_size=30522,
                         max_position_embeddings=512), 0),
    ("2048 positions", dict(num_hidden_layers=2, hidden_size=128, num_attention_heads=2, intermediate_size=512, vocab_size=30522,
                            max_position_embeddings=2048), 2048)])
def test_fp16_shapes(ctx, label, cfg, long_len):
    state = br.head_state(cfg, br.random_state(cfg, 13), 13)       # its position table has the config's rows
    enc = _encoder(ctx, cfg, state)
    g = np.random.default_rng(11)
    flat, toff, seg, poff = _random_pairs(g, 4, 10, d_len=(0, 200) if not long_len else (1900, 2600), max_length=long_len or 512)
    lens = np.diff(toff)
    assert not long_len or lens.max() == 2048
    idx = sorted(set(br.sample(lens.tolist(), 6).tolist()) | {int(lens.argmax())})
    _check_logits(label, cfg, state, enc, flat, toff, seg, poff, idx)
    enc.destroy()


@pytest.mark.gpu
def test_fp16_keeps_the_order_of_separated_scores_and_the_tie_rule(ctx):
    from kaito_b200 import _native
    from kaito_b200.rerank import build_pairs
    cfg = CE_MODELS["MiniLM-L6"]
    enc = _encoder(ctx, cfg, _state(cfg, "bench"))
    flat, toff, seg, poff = _random_pairs(np.random.default_rng(3), 32, 30)
    s32 = _all_scores(enc, flat, toff, seg, poff, _native.RERANK_SIGMOID)
    enc.set_precision("fp16")
    s16 = _all_scores(enc, flat, toff, seg, poff, _native.RERANK_SIGMOID)
    assert float(np.abs(s16 - s32).max()) <= SCORE_TOL_FP16
    checked = 0
    for q in range(32):
        a, b = s32[poff[q]:poff[q + 1]].astype(np.float64), s16[poff[q]:poff[q + 1]].astype(np.float64)
        far = np.abs(a[:, None] - a[None, :]) > 2 * SCORE_TOL_FP16
        assert ((a[:, None] > a[None, :]) == (b[:, None] > b[None, :]))[far].all(), q
        checked += int(far.sum())
    assert checked > 0
    # duplicate passages: exact ties, kept in position order (the constructed-tie case of test_selection_order_and_ties)
    n, top_k = 300, 10
    g = np.random.default_rng(n + top_k)
    qt = g.integers(1000, 30000, 8).astype(np.int32)
    uniq = [g.integers(1000, 30000, int(g.integers(1, 40))).astype(np.int32) for _ in range(n // 3)]
    cands = [uniq[int(g.integers(len(uniq)))] for _ in range(n)]
    flat, toff, seg, poff = build_pairs(2, 3, [(qt, 8)] * 3, [[(d, len(d)) for d in cands]] * 2 + [[]], 512)
    pos, sc = enc.rerank(poff, flat, toff, seg, top_k)
    full = _all_scores(enc, flat, toff, seg, poff[:2], _native.RERANK_SIGMOID)
    order = np.lexsort((np.arange(n), -full))[:top_k]
    assert len(set(full.tolist())) < n
    for qi in range(2):
        assert pos[qi].tolist() == order.tolist() and np.array_equal(sc[qi], full[order])
    assert (pos[2] == -1).all() and np.isnan(sc[2]).all()
    enc.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("cls_rows", [True, False])
def test_default_mode_is_untouched_by_a_switch_to_fp16_and_back(ctx, cls_rows):
    cfg = CE_MODELS["MiniLM-L6"]
    enc = _encoder(ctx, cfg, _state(cfg, "bench"))
    enc.debug_cls_rows(cls_rows)
    flat, toff, seg, poff = _random_pairs(np.random.default_rng(1), 16, 30)
    toks = [np.random.default_rng(i).integers(1000, 30000, 20 + i % 9).astype(np.int32) for i in range(64)]

    def run():      # three calls per shape: eager, capture, replay
        out = []
        for _ in range(3):
            out += [*enc.rerank(poff, flat, toff, seg, 10), enc.embed(toks)]
        return out
    first = run()
    enc.set_precision("fp16")
    half = run()
    enc.set_precision("fp32")
    third = run()
    for a, c in zip(first, third):
        assert np.array_equal(a, c, equal_nan=True)
    for k in range(3, 9):                                        # fp16 mode: the same bits eager, captured and replayed
        assert np.array_equal(half[k], half[k - 3], equal_nan=True)
    assert not np.array_equal(half[1], first[1]) and not np.array_equal(half[2], first[2])      # and it is another forward
    with pytest.raises(ValueError):
        enc.set_precision("bf16")
    enc.destroy()


@pytest.mark.gpu
def test_fp16_chunked_call_agrees_with_per_query_calls(ctx):
    """the construction of test_gpu_rerank's chunking test.  A query alone and a query inside a 65,536-token forward take
    different GEMM plans (tile width, K split), so scores agree within the mode's bound rather than bit for bit, as in the
    default mode"""
    cfg = CE_MODELS["MiniLM-L6"]
    enc = _encoder(ctx, cfg, _state(cfg, "bench"))
    enc.set_precision("fp16")
    flat, toff, seg, poff = _random_pairs(np.random.default_rng(9), 64, 30, q_len=(4, 20), d_len=(20, 80))
    assert toff[-1] > 65536
    pos, sc = enc.rerank(poff, flat, toff, seg, 10)
    for q in range(0, 64, 7):
        a, b = int(poff[q]), int(poff[q + 1])
        p1, s1 = enc.rerank(np.array([0, b - a], np.int32), flat[toff[a]:toff[b]], toff[a:b + 1] - toff[a], seg[a:b], 10)
        assert float(np.abs(s1[0] - sc[q]).max()) <= SCORE_TOL_FP16
        gaps = np.diff(-sc[q].astype(np.float64))
        for j in range(10):
            if (j == 0 or gaps[j - 1] > 2 * SCORE_TOL_FP16) and (j == 9 or gaps[j] > 2 * SCORE_TOL_FP16):
                assert p1[0, j] == pos[q, j], (q, j)
    enc.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("model,pooling", [("MiniLM-L12", "cls"), ("MiniLM-L6", "mean")])     # bge-small, all-MiniLM-L6-v2
def test_fp16_embeddings_within_torch_bf16(ctx, model, pooling):
    import bench
    from kaito_b200 import _native
    from tests.test_gpu_embed import _embedder
    cfg = CE_MODELS[model]
    state = bench.random_bert_state(cfg, 2)
    emb = _embedder(ctx, cfg, state)
    emb.set_pooling(_native.POOL_MEAN if pooling == "mean" else _native.POOL_CLS)
    emb.set_precision("fp16")
    g = np.random.default_rng(8)
    toks = [g.integers(1000, 30000, int(n)).astype(np.int32) for n in [1, 2, 17, 32, 64, 129, 300, 512] + g.integers(3, 200, 56).tolist()]
    got = emb.embed(toks)
    idx = br.sample([len(t) for t in toks], 16)
    ref = br.Fp64Bert(cfg, state)
    sub = [toks[i] for i in idx]
    c64, m64 = ref.pooled(sub)[:2]
    c16, m16 = _bf16_pools(ref, sub)
    e64, e16 = (m64, m16) if pooling == "mean" else (c64, c16)
    k5, t16 = float(np.abs(got[idx] - e64).max()), float(np.abs(e16 - e64).max())
    print(f"embed fp16 vs fp64 | {model} {pooling} | k5 {k5:.2e} | torch bf16 {t16:.2e} | ratio {k5 / t16:.3f} | "
          f"L2^2 dev {br.l2_deviation(got[idx], e64):.2e} | torch bf16 L2^2 dev {br.l2_deviation(e16, e64):.2e}")
    assert k5 <= t16, (k5, t16)
    emb.destroy()
