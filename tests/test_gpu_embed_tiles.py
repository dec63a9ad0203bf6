"""K5's GEMM tile widths and the [CLS]-rows-only last layer give the same bits as the paths they replace.

- 128 x 64 and 128 x 32 tiles against 128 x 128 tiles (the forward's choice at these M): every output element is summed
  over the same K steps of 16 in the same order into the same two accumulators, so the results are compared with ==, at
  the four bge-base GEMMs of the bench batch (256 x 32 tokens), bge-small's four and ragged M.
- CLS pooling with the last layer's O projection / FFN / LayerNorms on the [CLS] rows against the same forward over every
  token (krag_debug_embedder_cls_rows), on the final embeddings, eager and replayed from a captured graph, and a
  CLS -> mean -> CLS switch between forwards of one shape."""
import numpy as np
import pytest

BASE = dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=30522)

# (M, N, K, gelu, residual) as the forward runs them: QKV, O (+residual), FFN1 (+GELU), FFN2 (+residual)
SHAPES = [(8192, 2304, 768, False, False), (8192, 768, 768, False, True), (8192, 3072, 768, True, False),
          (8192, 768, 3072, False, True),
          (8192, 1152, 384, False, False), (8192, 384, 384, False, True), (8192, 1536, 384, True, False),
          (8192, 384, 1536, False, True),
          (8193, 2304, 768, False, False), (8191, 768, 3072, False, True), (1000, 1536, 384, True, False),
          (4100, 768, 768, False, True)]


def _operands(M, N, K, res, seed):
    g = np.random.default_rng(seed)
    A = g.standard_normal((M, K)).astype(np.float32)
    B = (g.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = g.standard_normal(N).astype(np.float32)
    R = g.standard_normal((M, N)).astype(np.float32) if res else None
    return A, B, bias, R


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,gelu,res", SHAPES)
def test_tile_widths_give_the_same_bits(ctx, M, N, K, gelu, res):
    from kaito_b200 import _native
    A, B, bias, R = _operands(M, N, K, res, M + 3 * N + 7 * K)
    picked = _native.debug_gemm_tf32(ctx, A, B, bias, R, gelu)
    for bn in (128, 64, 32):
        got = _native.debug_gemm_tf32(ctx, A, B, bias, R, gelu, tile_n=bn)
        assert np.array_equal(got, picked), (bn, np.abs(got - picked).max())


def _embedder(ctx, cfg, seed=0):
    import bench
    from kaito_b200 import _native
    e = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                         cfg["vocab_size"], 512)
    e.load_state_dict(bench.random_bert_state(cfg, seed))
    return e


@pytest.fixture(scope="module")
def base(ctx):
    e = _embedder(ctx, BASE)
    yield e
    e.destroy()


def _forwards(e, toks, n=3):
    """n forwards of one shape: eager, captured, replayed; all must agree"""
    outs = [e.embed(toks) for _ in range(n)]
    for o in outs[1:]:
        assert np.array_equal(o, outs[0])
    return outs[0]


def _cases():
    g = np.random.default_rng(7)
    bench_q = [np.random.default_rng(100 + b).integers(1000, 30000, 32) for b in range(256)]
    ragged = [g.integers(1000, 30000, int(n)) for n in np.concatenate([[1, 512, 2, 129], g.integers(1, 513, 20)])]
    return {"bench 256 x 32": bench_q, "ragged 1-512": ragged, "batch 1 x 300": [g.integers(1000, 30000, 300)]}


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["bench 256 x 32", "ragged 1-512", "batch 1 x 300"])
def test_cls_rows_last_layer_equals_full_layer(base, case):
    toks = _cases()[case]
    try:
        base.debug_cls_rows(False)
        full = _forwards(base, toks)
        base.debug_cls_rows(True)
        rows = _forwards(base, toks)
    finally:
        base.debug_cls_rows(True)
    assert np.array_equal(rows, full), np.abs(rows - full).max()


@pytest.mark.gpu
def test_pooling_switch_with_graph_replay(base):
    from kaito_b200 import _native
    toks = _cases()["ragged 1-512"]
    try:
        cls1 = _forwards(base, toks)
        base.set_pooling(_native.POOL_MEAN)
        mean = _forwards(base, toks)
        base.set_pooling(_native.POOL_CLS)
        cls2 = _forwards(base, toks)
        base.debug_cls_rows(False)
        cls_full = _forwards(base, toks)
    finally:
        base.set_pooling(_native.POOL_CLS)
        base.debug_cls_rows(True)
    assert np.array_equal(cls1, cls2) and np.array_equal(cls1, cls_full)
    # mean pooling ran the full last layer: the [CLS] rows cannot stand in for it
    long_rows = [i for i, t in enumerate(toks) if len(t) > 1]
    assert not np.allclose(mean[long_rows], cls1[long_rows], atol=1e-3)
