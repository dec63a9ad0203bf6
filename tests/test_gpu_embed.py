"""K5 (BERT encoder forward; linear layers on fp16 wgmma with split fp16 operands = fp32-accurate products) against
transformers.BertModel in fp64 on the CPU with the same weights (the real bge weights are not available offline; an opt-in
test at the bottom runs the reference's own golden when a local snapshot is given), CLS pooling + L2 norm as
sentence-transformers does for bge (embedding/huggingface_local_embedding.py:34-53).

Every forward case is held to two bounds (tests/bert_reference.py):
- the north_star contract: the L2^2 score against 64 random unit rows moves by less than 1e-4;
- the fp32 yardstick: K5's max |e - e64| over the checked sequences is at most F times torch fp32's max |e32 - e64| on the
  same sequences (floored at 2^-23).  F = 40: measured on an H100 80GB HBM3 (700 W power limit) over every forward case
  below, the ratio was at most 21.0 (bge-large, stressed weights, ragged queries), 12.3 with the bench's bge-large weights and
  at most 7.3 on the 1-2-layer models (DESIGN.md K5).  The ratio grows with depth and width: the tensor cores accumulate
  long K ranges less accurately than fp32 FMA chains.  Dropping a correction product or the online-softmax rescaling of
  the correction accumulator puts the 2-layer stressed cases at 57 or more.
Two weight regimes: "bench" = bench.random_bert_state, the weights bench.py times (N(0, 0.02), zero biases: near-uniform
attention); "stressed" = bert_reference.stressed_state (outlier hidden channels and attention scores of std ~12, so the
softmax is nearly one-hot).  Every forward case also asserts that no Linear input or output of the fp64 forward leaves the
split-fp16 operand range (< 6e4), so a failure here is K5's and not its input's."""
import numpy as np
import pytest

from tests import bert_reference as br

F = 40.0
REGIMES = ["bench", "stressed"]
BGE = {n: dict(c, max_position_embeddings=512) for n, c in __import__("bench").BGE.items()}
QUERY_TOKENS = 32                    # bench.py --query-tokens default


# --------------------------------------------------------------------------------------------------------------- helpers
def _state(cfg, regime, seed=0):
    """(weights, their fp64 reference)"""
    import bench
    if regime == "stressed":
        return br.stressed_state(cfg, seed)
    st = bench.random_bert_state(cfg, seed)
    return st, br.Fp64Bert(cfg, st)


def _embedder(ctx, cfg, state):
    from kaito_b200 import _native
    emb = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                           cfg["vocab_size"], cfg.get("max_position_embeddings", 512))
    emb.load_state_dict(state)
    return emb


def _reference(ref, toks):
    """fp64 and fp32 embeddings of the given sequences, and the largest Linear operand the fp64 forward saw"""
    ref.range_max = 0.0
    e64 = ref.embed(toks)
    return e64, ref.embed_fp32(toks), ref.range_max


def _assert_fp64(label, got, e64, e32, range_max):
    k5, t32, ratio = br.yardstick(got, e64, e32)
    l2 = br.l2_deviation(got, e64)
    print(f"K5 vs fp64 | {label} | k5 {k5:.2e} | L2^2 dev {l2:.2e} | torch fp32 {t32:.2e} | ratio {ratio:.2f} | "
          f"max Linear operand {range_max:.3g}")
    br.check_range(range_max)
    assert np.allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-5)
    assert l2 < 1e-4, (label, l2)                                   # the contract
    assert ratio <= F, (label, k5, t32, ratio)                      # and fp32-level arithmetic


def _bench_queries(B=256):
    return [np.random.default_rng(100 + b).integers(1000, 30000, QUERY_TOKENS) for b in range(B)]


def _check_batch(label, emb, ref, toks, n_sample=32, flat=False):
    """embed the whole batch on the GPU, compare a sample (bert_reference.sample) against fp64"""
    from kaito_b200 import _native
    got = emb.embed_flat(*_native.Embedder.pack(toks)) if flat else emb.embed(toks)
    idx = br.sample([len(t) for t in toks], n_sample)
    _assert_fp64(f"{label} ({len(toks)} seqs, {sum(len(t) for t in toks)} tok, {len(idx)} checked)", got[idx],
                 *_reference(ref, [toks[i] for i in idx]))
    return got


def _sample_rows(M, n=512, seed=0):
    """rows of an M-row GEMM checked against fp64: all of them up to 4096, else both ends, every tile boundary's
    neighbours near the ends and a random draw"""
    if M <= 4096:
        return np.arange(M)
    rows = set(range(128)) | set(range(M - 128, M)) | {127, 128, 129, 255, 256, 8191 % M, 8192 % M}
    rows |= set(np.random.default_rng(seed).choice(M, n, replace=False).tolist())
    return np.array(sorted(r for r in rows if r < M))


def _gelu(x):
    from scipy.special import erf
    return 0.5 * x * (1 + erf(x / np.sqrt(2)))


# ------------------------------------------------------------------------------------------------------------ raw GEMMs
@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,gelu,res", [(10, 128, 64, False, False), (300, 384, 384, False, True),
                                           (1000, 1152, 384, False, False), (257, 1536, 384, True, False),
                                           (129, 384, 1536, False, True), (4096, 768, 768, True, True),
                                           # small-M split-K path (128 x 32 tiles, M <= 128; 128 x 64 tiles above)
                                           (1, 768, 768, False, False), (16, 2304, 768, False, False), (16, 3072, 768, True, False),
                                           (100, 768, 3072, False, True), (128, 384, 384, False, True), (7, 1024, 4096, False, True),
                                           (512, 768, 768, False, True), (400, 768, 3072, False, True), (512, 2304, 768, False, False),
                                           (1024, 768, 3072, False, True), (600, 1024, 4096, False, False),
                                           # production M: bge-base's four layers over 256 x 32 query tokens, bge-small's QKV and
                                           # FFN1 over a 65,536-token index batch, and M one either side of a tile boundary
                                           (8192, 2304, 768, False, False), (8192, 768, 768, False, True),
                                           (8192, 3072, 768, True, False), (8192, 768, 3072, False, True),
                                           (65536, 1152, 384, False, False), (65536, 1536, 384, True, False),
                                           (8191, 2304, 768, False, False), (8193, 768, 3072, False, True)])
def test_gemm_tf32_matches_numpy(ctx, M, N, K, gelu, res):
    from kaito_b200 import _native
    g = np.random.default_rng(M + N + K)
    A = g.standard_normal((M, K)).astype(np.float32)
    B = (g.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = g.standard_normal(N).astype(np.float32)
    R = g.standard_normal((M, N)).astype(np.float32) if res else None
    got = _native.debug_gemm_tf32(ctx, A, B, bias, R, gelu)
    rows = _sample_rows(M)
    ref = A[rows].astype(np.float64) @ B.astype(np.float64).T + bias
    if gelu:
        ref = _gelu(ref)
    if res:
        ref = ref + R[rows]
    err = np.abs(got[rows] - ref)
    print(f"gemm {M}x{N}x{K}: max {err.max():.2e} mean {err.mean():.2e} over {len(rows)} rows")
    # |a.b| ~ 1: an fp32 SIMT GEMM is at ~sqrt(K) 2^-24 ~ 2e-6; the split-fp16 tensor-core product adds 2^-22 operand error
    # and the tensor core's own accumulation rounding (TF32 operands, which this replaced, sat at 2e-2 / 1e-3)
    assert err.max() < 5e-5 and err.mean() < 5e-6, (err.max(), err.mean())


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(8192, 2304, 768), (300, 1536, 384)])
def test_gemm_outlier_columns_matches_numpy(ctx, M, N, K):
    """BERT-like activations: a few columns of |a| ~ 1e3 among O(1) ones (the outlier features of trained BERTs).  The error
    is held relative to sum_k |a_k b_k|, the scale fp32 accumulation error grows with: fp32 SIMT sits near 2^-23 of it."""
    from kaito_b200 import _native
    g = np.random.default_rng(M + N + K + 1)
    A = g.standard_normal((M, K)).astype(np.float32)
    cols = g.choice(K, 4, replace=False)
    A[:, cols] = (g.choice([-1.0, 1.0], (M, 4)) * g.uniform(500.0, 2000.0, (M, 4))).astype(np.float32)
    B = (g.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = g.standard_normal(N).astype(np.float32)
    got = _native.debug_gemm_tf32(ctx, A, B, bias, None, False)
    rows = _sample_rows(M)
    A64, B64 = A[rows].astype(np.float64), B.astype(np.float64)
    ref = A64 @ B64.T + bias
    scale = np.abs(A64) @ np.abs(B64).T + np.abs(bias)
    rel = np.abs(got[rows] - ref) / scale
    print(f"gemm outliers {M}x{N}x{K}: max |a.b| {np.abs(ref).max():.3g}, max err/sum|ab| {rel.max():.2e}")
    assert rel.max() < 2.0 ** -18, rel.max()


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,res", [(16, 768, 3072, True), (1, 768, 768, True), (512, 384, 384, True), (300, 1024, 1024, False),
                                        (4096, 768, 768, True),
                                        (8192, 768, 768, True), (8192, 768, 3072, True), (65536, 384, 384, True),
                                        (65536, 384, 1536, True), (8191, 768, 768, True), (8193, 768, 3072, True)])
def test_linear_layernorm_matches_numpy(ctx, M, N, K, res):
    """GEMM + bias + residual + LayerNorm through the dispatcher (split-K reduce/LN kernel for few rows, fused epilogue +
    LN kernel otherwise) against fp64 numpy.  Tolerance: fp32-level products on |a.b| ~ 1 before a unit-variance LN."""
    from kaito_b200 import _native
    g = np.random.default_rng(M * 7 + N + K)
    A = g.standard_normal((M, K)).astype(np.float32)
    B = (g.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = g.standard_normal(N).astype(np.float32)
    R = g.standard_normal((M, N)).astype(np.float32) if res else None
    gamma, beta = (1 + 0.1 * g.standard_normal(N)).astype(np.float32), (0.1 * g.standard_normal(N)).astype(np.float32)
    got = _native.debug_linear_ln(ctx, A, B, bias, R, gamma, beta, 1e-12)
    rows = _sample_rows(M)
    y = A[rows].astype(np.float64) @ B.astype(np.float64).T + bias + (R[rows] if res else 0)
    ref = (y - y.mean(1, keepdims=True)) / np.sqrt(y.var(1, keepdims=True) + 1e-12) * gamma + beta
    err = np.abs(got[rows] - ref)
    print(f"linear+ln {M}x{N}x{K}: max {err.max():.2e} mean {err.mean():.2e} over {len(rows)} rows")
    assert err.max() < 5e-5 and err.mean() < 5e-6, (err.max(), err.mean())


# ------------------------------------------------------------------------------------------- the fp64 reference (CPU)
SMALL_2L = dict(num_hidden_layers=2, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=1000,
                max_position_embeddings=512)
BASE_2L = dict(SMALL_2L, hidden_size=768, intermediate_size=3072)


@pytest.mark.parametrize("regime", REGIMES)
def test_fp64_reference_alone_equals_padded_batch(regime):
    """The reference runs each sequence alone (K5 packs them without padding); in fp64 that is the padded, attention-masked
    batch forward to 1e-12, so checking a sample of sequences is checking the batch."""
    _, ref = _state(SMALL_2L, regime, seed=5)
    g = np.random.default_rng(5)
    toks = [g.integers(0, 1000, n) for n in (1, 7, 32, 33, 130, 257)]
    assert np.abs(ref.embed(toks) - ref.embed_padded(toks)).max() < 1e-12


def test_stressed_state_has_sharp_attention_and_outliers():
    """what the stressed regime promises: attention score std 8-16 in every layer, operands well inside the fp16 range"""
    st, ref = br.stressed_state(BASE_2L, seed=2)
    g = np.random.default_rng(2)
    toks = [g.integers(0, 1000, n) for n in (20, 64, 200)]
    stds = [ref.attention_score_std(toks, l) for l in range(BASE_2L["num_hidden_layers"])]
    ref.range_max = 0.0
    ref.embed(toks)
    print(f"stressed: score std {stds}, max Linear operand {ref.range_max:.3g}")
    assert all(8 <= s <= 16 for s in stds), stds
    assert 20 < ref.range_max < br.RANGE_LIMIT
    assert sum(float(st["embeddings.LayerNorm.weight"][c]) > 9 for c in range(BASE_2L["hidden_size"])) in (2, 3, 4)


def test_range_guard_fires_past_fp16():
    st = br.random_state(SMALL_2L, seed=1)
    toks = [np.arange(10)]
    ref = br.Fp64Bert(SMALL_2L, st)
    ref.embed(toks)
    br.check_range(ref.range_max)
    st["embeddings.LayerNorm.bias"][7] = 7.0e4            # LayerNorm output (the QKV GEMM's input) past 65504
    ref = br.Fp64Bert(SMALL_2L, st)
    ref.embed(toks)
    with pytest.raises(AssertionError, match="split-fp16 operand range"):
        br.check_range(ref.range_max)


# ------------------------------------------------------------------------------------------------ forward: small shapes
@pytest.mark.gpu
@pytest.mark.parametrize("name,cfg,lens", [
    ("small-2L", dict(num_hidden_layers=2, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=1000,
                      max_position_embeddings=512), [1, 3, 17, 64, 130, 512]),
    ("short-32", dict(num_hidden_layers=2, hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=900,
                      max_position_embeddings=512), [1, 5, 32, 31]),
    ("short-64", dict(num_hidden_layers=2, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=900,
                      max_position_embeddings=512), [33, 64, 7, 2]),
    ("short-64-large", dict(num_hidden_layers=1, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, vocab_size=900,
                            max_position_embeddings=512), [40, 64]),
    ("bge-small", dict(num_hidden_layers=12, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=2000,
                       max_position_embeddings=512), [9, 32, 200]),
    ("base-3L", dict(num_hidden_layers=3, hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=1500,
                     max_position_embeddings=512), [5, 33, 256]),
    ("large-2L", dict(num_hidden_layers=2, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, vocab_size=1200,
                      max_position_embeddings=512), [7, 128]),
])
def test_bert_forward_matches_transformers(ctx, name, cfg, lens):
    state = br.random_state(cfg, seed=len(name))
    g = np.random.default_rng(3)
    toks = [g.integers(0, cfg["vocab_size"], n).tolist() for n in lens]
    emb = _embedder(ctx, cfg, state)
    try:
        got = emb.embed(toks)
        e64, e32, rng = _reference(br.Fp64Bert(cfg, state), toks)
        _assert_fp64(name, got, e64, e32, rng)
        # batching changes only the summation order (packed, no padding; the GEMM tiling and split-K factor follow the
        # token count, as torch's own kernels do): alone, a sequence meets the same bound
        alone = emb.embed([toks[-1]])
        _assert_fp64(f"{name} last alone", alone, e64[-1:], e32[-1:], rng)
        assert np.array_equal(emb.embed([toks[-1]])[0], alone[0])          # same shape -> same bits
    finally:
        emb.destroy()


# --------------------------------------------------------------------------------------- forward: the shapes that run
@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("model", ["bge-small", "bge-base", "bge-large"])
def test_query_batch_matches_fp64(ctx, model, regime):
    """bench.py's query step: 256 queries x 32 tokens (its token recipe) through every layer; and a ragged 256-query batch of
    12-48 tokens (the bge instruction prefix puts real queries there), whose max_len in (32, 64] selects the 64-key
    attention variant."""
    cfg = BGE[model]
    state, ref = _state(cfg, regime)
    emb = _embedder(ctx, cfg, state)
    try:
        _check_batch(f"{model} {regime} 256x32", emb, ref, _bench_queries())
        g = np.random.default_rng(7)
        ragged = [g.integers(1000, 30000, n) for n in g.integers(12, 49, 256)]
        assert 32 < max(len(t) for t in ragged) <= 64
        _check_batch(f"{model} {regime} 256 ragged 12-48", emb, ref, ragged)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_index_batch_small_matches_fp64(ctx, regime):
    """/index on bge-small: 65,536 tokens (128 x 512) through embed_flat, the service's call
    (GpuBertEmbedding.max_batch_tokens), and a ragged batch of 1-512 tokens up to 65,536 in total.  The ragged batch also
    carries queries of the bench's 256-query batch: each is held to the fp64 bound alone, inside the 256-query batch and
    inside the 64k-token batch."""
    from kaito_b200 import _native
    cfg = BGE["bge-small"]
    state, ref = _state(cfg, regime)
    emb = _embedder(ctx, cfg, state)
    try:
        g = np.random.default_rng(11)
        _check_batch(f"bge-small {regime} 128x512", emb, ref, [g.integers(1000, 30000, 512) for _ in range(128)], n_sample=20, flat=True)

        queries = _bench_queries()
        picked = [0, 3, 4, 127, 128, 255]
        ragged, at, total = [], [], 0
        while True:
            if len(ragged) % 37 == 5 and len(at) < len(picked):       # plant the queries between documents
                t = queries[picked[len(at)]]
                at.append(len(ragged))
            else:
                t = g.integers(1000, 30000, int(g.integers(1, 513)))
            if total + len(t) > 65536:
                break
            ragged.append(t); total += len(t)
        assert len(at) == len(picked) and total > 65000
        got_r = _check_batch(f"bge-small {regime} ragged 1-512", emb, ref, ragged, n_sample=24, flat=True)

        e64, e32, rng = _reference(ref, [queries[i] for i in picked])
        alone = np.concatenate([emb.embed([queries[i]]) for i in picked])
        in_batch = emb.embed_flat(*_native.Embedder.pack(queries))[picked]
        _assert_fp64(f"bge-small {regime} queries alone", alone, e64, e32, rng)
        _assert_fp64(f"bge-small {regime} queries in 256x32", in_batch, e64, e32, rng)
        _assert_fp64(f"bge-small {regime} queries in 64k ragged", got_r[at], e64, e32, rng)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_index_batch_base_matches_fp64(ctx, regime):
    """bge-base at 32 x 512: head dim 64 over 8 double-buffered 64-key blocks (attention_mma_kernel<64, 4, 64, 2>)"""
    cfg = BGE["bge-base"]
    state, ref = _state(cfg, regime)
    emb = _embedder(ctx, cfg, state)
    try:
        g = np.random.default_rng(13)
        _check_batch(f"bge-base {regime} 32x512", emb, ref,
                     [g.integers(1000, 30000, 512) for _ in range(32)], n_sample=8)
    finally:
        emb.destroy()


EDGE_LENS = [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512]


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("cfg", [SMALL_2L, BASE_2L], ids=["dh32", "dh64"])
def test_attention_key_block_edges(ctx, cfg, regime):
    """Every sequence checked: lengths at each side of the 16-row query and 32 / 64-key block boundaries in one batch (the
    short ones then share the double-buffered launch), and batches whose max_len is exactly 32, 33, 64 and 65, so each
    attention variant and its neighbour run at their limits."""
    state, ref = _state(cfg, regime, seed=17)
    emb = _embedder(ctx, cfg, state)
    try:
        g = np.random.default_rng(17)
        batches = [EDGE_LENS] + [[m, 1, m - 1, 16, m] for m in (32, 33, 64, 65)]
        for lens in batches:
            toks = [g.integers(0, cfg["vocab_size"], n) for n in lens]
            _assert_fp64(f"dh{cfg['hidden_size'] // 12} {regime} lens {lens}", emb.embed(toks), *_reference(ref, toks))
    finally:
        emb.destroy()


# ------------------------------------------------------------------------------------------- device output and graphs
def _small_embedder(ctx, seed=21):
    state = br.random_state(SMALL_2L, seed)
    return _embedder(ctx, SMALL_2L, state), state


@pytest.mark.gpu
def test_embed_dev_layout_and_write_after_read(ctx):
    """krag_embed_dev writes rows of stride ld_out into the caller's buffer, makes the caller's stream wait for them, and its
    final kernel waits for work the caller enqueued on that stream before the call (the previous batch still reading the
    buffer): the consumer here sleeps ~50 ms and then copies the buffer, so without that wait the copy would see the new rows."""
    import torch
    from kaito_b200 import _native
    emb, _ = _small_embedder(ctx)
    try:
        d, B = SMALL_2L["hidden_size"], 5
        ld = d + 32
        g = np.random.default_rng(23)
        lens = [3, 9, 1, 20, 7]
        toks1 = [g.integers(0, 1000, n) for n in lens]
        toks2 = [g.integers(0, 1000, n) for n in lens]
        want1, want2 = emb.embed(toks1), emb.embed(toks2)
        buf = torch.full((B + 3, ld), float("nan"), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        emb.embed_dev(*_native.Embedder.pack(toks1), buf.data_ptr(), ld, s.cuda_stream)
        with torch.cuda.stream(s):
            snap = buf.clone()
        s.synchronize()
        got = snap.cpu().numpy()
        assert np.array_equal(got[:B, :d], want1)
        assert np.isnan(got[:B, d:]).all() and np.isnan(got[B:]).all()

        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)            # ~50 ms of clock cycles
            old = buf.clone()
        emb.embed_dev(*_native.Embedder.pack(toks2), buf.data_ptr(), ld, s.cuda_stream)
        with torch.cuda.stream(s):
            new = buf.clone()
        s.synchronize()
        assert np.array_equal(old.cpu().numpy()[:B, :d], want1), "the embeddings overwrote rows the consumer was still reading"
        assert np.array_equal(new.cpu().numpy()[:B, :d], want2)
    finally:
        emb.destroy()


@pytest.mark.gpu
def test_embed_into_rows(ctx):
    """ShardedRetriever.embed_into (world 1) on an index at the bench's dim: the rows are embed()'s, bit for bit; a row
    layout wider than the model (corpus dim above the embedding dim) gets zero padding columns"""
    import torch
    from kaito_b200 import _native
    from kaito_b200.sharded import NativeStages, ShardedRetriever
    cfg = BASE_2L
    d = cfg["hidden_size"]
    emb = _embedder(ctx, cfg, br.random_state(cfg, 29))
    ix = ctx.create_index("embed_into", d)
    try:
        g = np.random.default_rng(29)
        ix.add(np.arange(100, dtype=np.uint64), g.standard_normal((100, d)).astype(np.float32))
        stages = NativeStages(ctx, ix)
        toks = [g.integers(0, 1000, n) for n in g.integers(1, 40, 12)]
        want = emb.embed(toks)
        flat, off = _native.Embedder.pack(toks)
        for dpad in (stages.dim_padded(), d + 32):
            sr = ShardedRetriever(stages, torch.device("cuda", 0), dpad)
            q = torch.full((len(toks), dpad), float("nan"), dtype=torch.float32, device="cuda")
            sr.embed_into(emb, flat, off, q)
            got = q.cpu().numpy()
            assert np.array_equal(got[:, :d], want), dpad
            assert (got[:, d:] == 0).all(), dpad
    finally:
        ix.drop()
        emb.destroy()


@pytest.mark.gpu
def test_graph_replay_matches_fresh_eager(ctx):
    """A forward is captured into a CUDA graph on the second call of its (n_tok, batch, max_len) and replayed after that.
    Eager, capture and replays with new tokens and the lengths permuted under the same key must each equal a fresh
    embedder's eager forward bit for bit; so must the key after the workspaces grew, and after more than 64 shapes
    dropped every graph."""
    emb, state = _small_embedder(ctx)
    g = np.random.default_rng(31)

    def fresh(toks):
        e = _embedder(ctx, SMALL_2L, state)
        try:
            return e.embed(toks)
        finally:
            e.destroy()

    def check_key(tag, n_calls=4):
        for i in range(n_calls):
            toks = [g.integers(0, 1000, n) for n in g.permutation([5, 3, 13, 8])]   # key (29, 4, 13)
            assert np.array_equal(emb.embed(toks), fresh(toks)), (tag, i)

    try:
        check_key("eager, capture, replay, replay")
        big = [g.integers(0, 1000, 64) for _ in range(40)]                # grows the workspaces: graphs and counts dropped
        assert np.array_equal(emb.embed(big), fresh(big))
        check_key("after growing", 3)
        for n in range(1, 67):                                            # 66 new keys, each captured: the 64-graph cap
            toks = [g.integers(0, 1000, n)]
            first = emb.embed(toks)
            assert np.array_equal(emb.embed(toks), first), n
        check_key("after the graph cap", 3)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.skipif(not __import__("os").environ.get("KRAG_MODEL_DIR"), reason="opt-in: KRAG_MODEL_DIR=<local BAAI/bge-small-en-v1.5 snapshot>")
def test_real_weights_reference_golden(ctx):
    """The one numeric golden the reference's own tests hold for this path (presets/ragengine/tests/api/test_main.py:159-164):
    after indexing "This is a test document" / updating it to "This is an updated test document", the chat query
    "updates test query" gets source_nodes[0].score == 0.48061275482177734 (rel 1e-6) -- the squared L2 distance between the
    bge-small-en-v1.5 embeddings of the query and of that document (faiss IndexFlatL2, faiss_store.py:44-49).  Needs the real
    checkpoint (not available offline): point KRAG_MODEL_DIR at a snapshot holding config.json, vocab.txt and
    model.safetensors / pytorch_model.bin."""
    import os
    from kaito_b200.embedding import GpuBertEmbedding
    emb = GpuBertEmbedding.from_pretrained(ctx, os.environ["KRAG_MODEL_DIR"])
    try:
        q = np.asarray(emb.get_query_embedding("updates test query"), np.float64)
        d = np.asarray(emb.get_text_embedding_batch(["This is an updated test document"])[0], np.float64)
        assert float(((q - d) ** 2).sum()) == pytest.approx(0.48061275482177734, rel=1e-4)   # 1e-4: north_star tolerance
    finally:
        emb._emb.destroy()
