"""K5 against fp64 across the encoder shapes it accepts (check_bert_config, embedder_create): hidden sizes 128 ... 1024 in
steps of 128, so mean pooling's G = hidden / 128 runs 1 ... 8; heads of 32 and of 64 dims at most widths; intermediate sizes
other than 4 x hidden, so FFN2 runs over 2 ... 64 k-blocks; position tables of 1024 and 2048 rows, so attention runs over up
to 32 key blocks.  The Google BERT miniatures (bert_uncased_L-*_H-*_A-*) and models with long position tables are in this
space.  Every case is held to the bounds of tests/test_gpu_embed.py: the L2^2 score against 64 unit rows moves by less
than 1e-4, the error is at most F = 40 times torch fp32's own, and no Linear operand of the fp64 forward leaves the
split-fp16 range.  The CLS row and the token mean are both taken from one fp64 forward per checked sequence.

Weights: "random" = bert_reference.random_state (non-zero biases and LayerNorm parameters; its position table has the
config's max_position_embeddings rows), "stressed" = bert_reference.stressed_state.  The batches of every case:
- Q: the bench's 256 queries x 32 tokens (the 128 x 128 / 128 x 64 GEMM plans, the [CLS]-rows last layer);
- F: 1, 3 and 17 sequences inside one 128-row tile (128 x 32 tiles, split-K, LayerNorm in splitk_reduce_kernel);
- R: the lengths of EDGE_LENS (1 ... 512) in one batch, so each attention variant runs;
- L: past 512 positions, up to max_position_embeddings, among short sequences (long cases only).
Also exact: the [CLS]-rows last layer gives the full layer's bits on Q; eager, captured and replayed forwards agree on F.
The cross-encoder (pooler GEMM, classifier_head_kernel) runs at every width, and the tensor sizes of a state must match
the config at finalize."""
import numpy as np
import pytest

from tests import bert_reference as br
from tests.test_gpu_embed import EDGE_LENS, _assert_fp64, _bench_queries, _embedder
from tests.test_gpu_rerank import F, SCORE_TOL, _all_scores, _encoder, _pairs_of, _random_pairs


def _cfg(layers, hidden, heads, inter, max_pos=512):
    return dict(num_hidden_layers=layers, hidden_size=hidden, num_attention_heads=heads, intermediate_size=inter,
                vocab_size=30522, max_position_embeddings=max_pos)


CASES = {  # name: BertConfig (the comment: what the case reaches that the bge / MiniLM / e5 shapes do not)
    "tiny": _cfg(2, 128, 2, 512),              # bert_uncased_L-2_H-128_A-2: G = 1, LayerNorm with half the lanes idle
    "tiny-dh32": _cfg(2, 128, 4, 128),         # dh 32 at 4 heads; FFN2 over K = 128 (2 k-blocks)
    "mini": _cfg(4, 256, 4, 1024),             # bert_uncased_L-4_H-256_A-4: G = 2
    "mini-dh32": _cfg(2, 256, 8, 640),         # FFN2 over 10 k-blocks
    "small-6h": _cfg(2, 384, 6, 1152),         # dh 64 at 384; FFN2 over 18 k-blocks
    "small": _cfg(4, 512, 8, 2048),            # bert_uncased_L-4_H-512_A-8: G = 4, FFN2 K = 2048 (128-wide tiles)
    "w512-dh32": _cfg(2, 512, 16, 896),        # FFN2 over 14 k-blocks
    "w640": _cfg(2, 640, 10, 2560),            # G = 5; the last LayerNorm lane group partial
    "w640-dh32": _cfg(2, 640, 20, 640),
    "w896": _cfg(2, 896, 14, 3584),            # G = 7
    "w896-dh32": _cfg(2, 896, 28, 1152),
    "base-dh32": _cfg(2, 768, 24, 3072),       # 24 heads
    "large-dh32": _cfg(1, 1024, 32, 4096),     # 32 heads
    "long-384": _cfg(2, 384, 12, 1536, 2048),  # dh 32 over up to 32 key blocks
    "long-768": _cfg(2, 768, 12, 3072, 1024),  # dh 64 over up to 16 key blocks
}
STRESSED = ("tiny", "w640", "w896", "long-384", "long-768")
N_SAMPLE = 24                                  # sequences checked against fp64 per batch (bert_reference.sample)
F_LENS = {"F1": [48], "F3": [64, 1, 33], "F17": list(range(1, 14)) + [8, 7, 6, 5]}


def batch_lengths(cfg):
    """batch name -> the sequence lengths of that batch, for one case"""
    out = {"Q": [32] * 256, **F_LENS, "R": list(EDGE_LENS)}
    mp = cfg["max_position_embeddings"]
    if mp > 512:
        out["L"] = [511, 1, 512, 5, 513, 575, 33, 576, 577, 1000, 64, mp - 1, 2, mp]
    return out


def _batches(cfg, seed):
    g = np.random.default_rng(seed)
    return {name: _bench_queries() if name == "Q" else [g.integers(1000, 30000, n) for n in lens]
            for name, lens in batch_lengths(cfg).items()}


def _forwards(emb, flat, off, n):
    """n forwards of one shape (the first eager, the second captured, then replays): all the same bits"""
    outs = [emb.embed_flat(flat, off) for _ in range(n)]
    for o in outs[1:]:
        assert np.array_equal(o, outs[0]), np.abs(o - outs[0]).max()
    return outs[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name,regime", [(n, "random") for n in CASES] + [(n, "stressed") for n in STRESSED])
def test_shape_matches_fp64(ctx, name, regime):
    from kaito_b200 import _native
    cfg = CASES[name]
    if regime == "stressed":
        state, ref = br.stressed_state(cfg, 11)
    else:
        state = br.random_state(cfg, 11)
        ref = br.Fp64Bert(cfg, state)
    emb = _embedder(ctx, cfg, state)
    try:
        for label, toks in _batches(cfg, 11).items():
            flat, off = _native.Embedder.pack(toks)
            n_calls = 3 if label.startswith("F") else 1
            cls = _forwards(emb, flat, off, n_calls)
            if label == "Q":
                try:
                    emb.debug_cls_rows(False)
                    full = emb.embed_flat(flat, off)
                finally:
                    emb.debug_cls_rows(True)
                assert np.array_equal(cls, full), np.abs(cls - full).max()
            emb.set_pooling(_native.POOL_MEAN)
            try:
                mean = _forwards(emb, flat, off, n_calls)
            finally:
                emb.set_pooling(_native.POOL_CLS)
            lens = [len(t) for t in toks]
            idx = br.sample(lens, N_SAMPLE)
            c64, m64, c32, m32, rng = ref.pooled([toks[i] for i in idx])
            what = f"{name} {regime} {label} ({len(toks)} seqs, {sum(lens)} tok, max {max(lens)}, {len(idx)} checked)"
            _assert_fp64(f"cls {what}", cls[idx], c64, c32, rng)
            _assert_fp64(f"mean {what}", mean[idx], m64, m32, rng)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_cross_encoder_matches_fp64(ctx, name):
    """4 queries x 30 pairs of up to 200 tokens, one call (the long cases: passages cut to pairs of max_position_embeddings
    tokens); then a query with one short pair alone, whose forward saves no tile: its [CLS] row is gathered from the full
    last layer"""
    from kaito_b200 import _native
    from kaito_b200.rerank import build_pairs
    cfg = CASES[name]
    mp = cfg["max_position_embeddings"]
    state = br.head_state(cfg, br.random_state(cfg, 13), 13)
    enc = _encoder(ctx, cfg, state)
    try:
        g = np.random.default_rng(13)
        flat, toff, seg, poff = _random_pairs(g, 4, 30, d_len=(0, 200) if mp == 512 else (0, mp + 300), max_length=mp)
        logit = _all_scores(enc, flat, toff, seg, poff, _native.RERANK_IDENTITY)
        score = _all_scores(enc, flat, toff, seg, poff, _native.RERANK_SIGMOID)
        lens = np.diff(toff)
        idx = sorted(set(br.sample(lens.tolist(), N_SAMPLE).tolist()) | set(np.flatnonzero(lens == mp)[:2].tolist()))
        if mp > 512:
            assert lens.max() == mp
        pairs = _pairs_of(flat, toff, seg, idx)
        got_l, got_s = logit[idx].astype(np.float64), score[idx].astype(np.float64)

        one = build_pairs(2, 3, [(g.integers(1000, 30000, 5).astype(np.int32), 5)],
                          [[(g.integers(1000, 30000, 20).astype(np.int32), 20)]], mp)
        one_l = _all_scores(enc, *one, _native.RERANK_IDENTITY)
        one_s = _all_scores(enc, *one, _native.RERANK_SIGMOID)
        pairs += _pairs_of(one[0], one[1], one[2], [0])
        got_l = np.append(got_l, one_l); got_s = np.append(got_s, one_s)

        l64, l32 = br.Fp64CrossEncoder(cfg, state).logits(pairs)
        k5, t32 = float(np.abs(got_l - l64).max()), float(np.abs(l32 - l64).max())
        ratio = k5 / max(t32, 2.0 ** -23)
        ds = float(np.abs(got_s - 1.0 / (1.0 + np.exp(-l64))).max())
        print(f"rerank vs fp64 | {name} | {len(pairs)} of {len(lens) + 1} pairs, longest {max(len(p[0]) for p in pairs)} tok | "
              f"logit err {k5:.2e} | torch fp32 {t32:.2e} | ratio {ratio:.2f} | sigmoid err {ds:.2e}")
        assert ratio <= F, (name, k5, t32, ratio)
        assert ds <= SCORE_TOL, (name, ds)
    finally:
        enc.destroy()


# ------------------------------------------------------------------------------------ tensor sizes against the config
SIZED = dict(num_hidden_layers=1, hidden_size=128, num_attention_heads=2, intermediate_size=256, vocab_size=1000,
             max_position_embeddings=1024)


@pytest.mark.gpu
def test_tensor_sizes_must_match_the_config(ctx):
    """Every encoder tensor with one row too few and one too many (a vector: one element) is refused at finalize with
    KRAG_E_INVALID and a message naming it: the kernels index the tables and weights by the config's sizes (a position
    table of 512 rows under max_position_embeddings 1024 would be read past its end).  No forward runs on such a state.
    A correct state loaded into the same embedder afterwards finalizes and embeds as a fresh embedder does."""
    from kaito_b200 import _native
    state = br.random_state(SIZED, 17)
    emb = _native.Embedder(ctx, 1, 128, 2, 256, 1000, 1024)
    try:
        for name, a in state.items():
            for delta in (-1, 1):
                rows = a.shape[0] + delta
                bad = dict(state)
                bad[name] = np.resize(a, (rows,) + a.shape[1:]).astype(np.float32)
                with pytest.raises(_native.KragError) as e:
                    emb.load_state_dict(bad)
                assert e.value.code == _native.KRAG_E_INVALID, (name, delta)
                assert f"{name} must hold {a.size} elements" in str(e.value), (name, delta, str(e.value))
        emb.load_state_dict(state)
        g = np.random.default_rng(17)
        toks = [g.integers(0, 1000, n) for n in (1, 40, 513, 1024)]
        fresh = _embedder(ctx, SIZED, state)
        try:
            want = fresh.embed(toks)
        finally:
            fresh.destroy()
        assert np.array_equal(emb.embed(toks), want)
    finally:
        emb.destroy()
