"""K5 (BERT encoder forward; linear layers on fp16 wgmma with split fp16 operands = fp32-accurate products) against
transformers.BertModel in fp32 on the CPU with the same seeded random weights (the real bge weights are not available
offline; an opt-in test at the bottom runs the reference's own golden when a local snapshot is given), CLS pooling + L2 norm
as sentence-transformers does for bge (embedding/huggingface_local_embedding.py:34-53).  Tolerances are written out: the
north_star contract is 1e-4 on the returned L2^2 scores; the embeddings themselves agree to a few 1e-6."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K,gelu,res", [(10, 128, 64, False, False), (300, 384, 384, False, True),
                                           (1000, 1152, 384, False, False), (257, 1536, 384, True, False),
                                           (129, 384, 1536, False, True), (4096, 768, 768, True, True),
                                           # small-M split-K path (128 x 32 tiles, M <= 128; 128 x 64 tiles above)
                                           (1, 768, 768, False, False), (16, 2304, 768, False, False), (16, 3072, 768, True, False),
                                           (100, 768, 3072, False, True), (128, 384, 384, False, True), (7, 1024, 4096, False, True),
                                           (512, 768, 768, False, True), (400, 768, 3072, False, True), (512, 2304, 768, False, False),
                                           (1024, 768, 3072, False, True), (600, 1024, 4096, False, False)])
def test_gemm_tf32_matches_numpy(ctx, M, N, K, gelu, res):
    from kaito_b200 import _native
    g = np.random.default_rng(M + N + K)
    A = g.standard_normal((M, K)).astype(np.float32)
    B = (g.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = g.standard_normal(N).astype(np.float32)
    R = g.standard_normal((M, N)).astype(np.float32) if res else None
    got = _native.debug_gemm_tf32(ctx, A, B, bias, R, gelu)
    ref = A.astype(np.float64) @ B.astype(np.float64).T + bias
    if gelu:
        from math import erf
        ref = 0.5 * ref * (1 + np.vectorize(erf)(ref / np.sqrt(2)))
    if res:
        ref = ref + R
    err = np.abs(got - ref)
    print(f"gemm {M}x{N}x{K}: max {err.max():.2e} mean {err.mean():.2e}")
    # |a.b| ~ 1: an fp32 SIMT GEMM is at ~sqrt(K) 2^-24 ~ 2e-6; the split-fp16 tensor-core product adds 2^-22 operand error
    # and the tensor core's own accumulation rounding (TF32 operands, which this replaced, sat at 2e-2 / 1e-3)
    assert err.max() < 5e-5 and err.mean() < 5e-6, (err.max(), err.mean())


@pytest.mark.parametrize("M,N,K,res", [(16, 768, 3072, True), (1, 768, 768, True), (512, 384, 384, True), (300, 1024, 1024, False),
                                        (4096, 768, 768, True)])
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
    y = A.astype(np.float64) @ B.astype(np.float64).T + bias + (R if res else 0)
    ref = (y - y.mean(1, keepdims=True)) / np.sqrt(y.var(1, keepdims=True) + 1e-12) * gamma + beta
    err = np.abs(got - ref)
    print(f"linear+ln {M}x{N}x{K}: max {err.max():.2e} mean {err.mean():.2e}")
    assert err.max() < 5e-5 and err.mean() < 5e-6, (err.max(), err.mean())


def _torch_reference(cfg, state, token_lists):
    import torch
    from transformers import BertConfig, BertModel
    m = BertModel(BertConfig(**cfg), add_pooling_layer=False).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()}, strict=False)
    out = []
    with torch.no_grad():
        for t in token_lists:
            h = m(input_ids=torch.tensor([t])).last_hidden_state[0, 0]
            out.append(torch.nn.functional.normalize(h, dim=0).numpy())
    return np.stack(out)


def _random_state(cfg, seed):
    import torch
    from transformers import BertConfig, BertModel
    torch.manual_seed(seed)
    m = BertModel(BertConfig(**cfg), add_pooling_layer=False)
    # default init is N(0, 0.02): give LayerNorm/bias non-trivial values so every term of the forward is exercised
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("bias"):
                p.normal_(0, 0.05)
            elif "LayerNorm.weight" in n:
                p.normal_(1.0, 0.1)
            elif p.dim() == 2 and "embeddings" not in n:
                p.normal_(0, 0.06)
    return {k: v.detach().numpy().astype(np.float32) for k, v in m.state_dict().items()}


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
    from kaito_b200 import _native
    state = _random_state(cfg, seed=len(name))
    g = np.random.default_rng(3)
    toks = [g.integers(0, cfg["vocab_size"], n).tolist() for n in lens]
    emb = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"],
                           cfg["intermediate_size"], cfg["vocab_size"], cfg["max_position_embeddings"])
    try:
        emb.load_state_dict(state)
        got = emb.embed(toks)
        ref = _torch_reference(cfg, state, toks)
        assert np.allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-5)
        cos = (got * ref).sum(1)
        dmax = np.abs(got - ref).max()
        # what /retrieve returns is L2^2 between this embedding and corpus rows: north_star tolerance 1e-4 on that score
        y = g.standard_normal((64, got.shape[1])).astype(np.float32)
        y /= np.linalg.norm(y, axis=1, keepdims=True)
        l2_got = ((got[:, None, :].astype(np.float64) - y[None]) ** 2).sum(-1)
        l2_ref = ((ref[:, None, :].astype(np.float64) - y[None]) ** 2).sum(-1)
        l2_dev = np.abs(l2_got - l2_ref).max()
        print(f"{name}: max|d| {dmax:.2e}  1-cos {1 - cos.min():.2e}  max L2^2 deviation {l2_dev:.2e}")
        assert l2_dev < 1e-4, l2_dev                       # the contract
        assert dmax < 2e-5 and cos.min() > 1 - 1e-6, (dmax, cos)   # and with margin: fp32-level agreement (TF32 was 5e-3 / 1e-4)
        # batching must not change a sequence's embedding beyond fp32 summation order (packed, no padding; the GEMM tiling
        # and split-K factor follow the token count, as torch's own kernels do)
        alone = emb.embed([toks[-1]])
        assert np.abs(alone[0] - got[-1]).max() < 2e-4 and float(alone[0] @ got[-1]) > 0.999999
        assert np.array_equal(emb.embed([toks[-1]])[0], alone[0])          # same shape -> same bits
    finally:
        emb.destroy()



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
