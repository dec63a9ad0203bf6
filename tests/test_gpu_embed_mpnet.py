"""K5 as an MPNet encoder (all-mpnet-base-v2, multi-qa-mpnet-base-*): the BERT forward plus a learned per-head bias on every
attention score, indexed by the bucket of the key - query distance (attention_mma_kernel's REL instantiations), positions
from row 2, no token-type table.  Held to the bounds of tests/test_gpu_embed.py against transformers.MPNetModel in fp64,
mean- or CLS-pooled and normalised in numpy: the L2^2 score against 64 unit rows moves by less than 1e-4 and the error is at
most F = 40 times torch fp32's own.  Two weight regimes: "bench" = bench.random_bert_state with a N(0, 1) bias table;
"stressed" = bert_reference.stressed_state (outlier channels, attention scores of std ~12) with a bias table of std 16 on a
third of the heads, which then dominates those heads' softmax.  Trained tables' magnitudes are not checked here: no
checkpoint is available offline.  Also: CLS-rows shortcut, device / host output and graph replay give the same bits; a
zeroed table moves the embeddings far past the bound; a wrong-sized table is refused naming it; fp16 mode stays within
torch bf16 autocast's error; an MPNet snapshot goes through GpuBertEmbedding.from_pretrained and a VectorStore /retrieve."""
import copy

import numpy as np
import pytest

from kaito_b200 import embedding as E
from tests import bert_reference as br
from tests import st_snapshot as sn
from tests.test_gpu_embed import _assert_fp64, _bench_queries

MPNET_BASE = dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=30527,
                  max_position_embeddings=514, layer_norm_eps=1e-5)          # all-mpnet-base-v2, multi-qa-mpnet-base-*
TWO_LAYER = dict(MPNET_BASE, num_hidden_layers=2)
HEAD32 = dict(MPNET_BASE, num_hidden_layers=2, hidden_size=384, intermediate_size=1536)   # head dim 32, hidden 384
REGIMES = ["bench", "stressed"]
_TO_MPNET = tuple((b, a) for a, b in E._MPNET_NAMES)


def _mpnet_name(k):
    for a, b in _TO_MPNET:
        k = k.replace(a, b)
    return k


def _state(cfg, regime, seed=0):
    """K5-named weights (BERT names, the zero token-type row, the bias table) of an MPNet encoder"""
    import bench
    g = np.random.default_rng(seed + 500)
    d, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    bcfg = dict(cfg, type_vocab_size=2)
    if regime == "stressed":
        st = br.stressed_state(bcfg, seed)[0]
        std = np.where(np.arange(heads) % 3 == 0, 16.0, 1.0)
    else:
        st = bench.random_bert_state(bcfg, seed)
        std = np.ones(heads)
    st["embeddings.position_embeddings.weight"] = (0.02 * g.standard_normal((cfg["max_position_embeddings"], d))).astype(np.float32)
    st["embeddings.token_type_embeddings.weight"] = np.zeros((1, d), np.float32)
    st[E.MPNET_REL_BIAS] = (g.standard_normal((32, heads)) * std).astype(np.float32)
    return st


class Fp64MPNet:
    """transformers.MPNetModel in fp64 and its fp32 twin, with bert_reference's Linear range hooks"""

    def __init__(self, cfg, state):
        import torch
        from transformers import MPNetConfig, MPNetModel
        from transformers.initialization import no_init_weights
        with no_init_weights():
            self.m64 = MPNetModel(MPNetConfig(**cfg, relative_attention_num_buckets=32), add_pooling_layer=False).double().eval()
        sd = {_mpnet_name(k): torch.from_numpy(np.asarray(v, np.float64)) for k, v in state.items() if "token_type" not in k}
        missing, unexpected = self.m64.load_state_dict(sd, strict=False)
        assert not missing and not unexpected, (missing, unexpected)
        self.m32 = copy.deepcopy(self.m64).float()
        self.range_max = 0.0
        for mod in self.m64.modules():
            if isinstance(mod, torch.nn.Linear):
                mod.register_forward_hook(lambda m, i, o: setattr(self, "range_max", max(self.range_max, float(i[0].abs().max()),
                                                                                        float(o.abs().max()))))

    def __call__(self, toks, pooling):
        """(fp64 embeddings, fp32 embeddings, largest Linear operand of the fp64 forward) of each sequence run alone"""
        self.range_max = 0.0
        c64, m64 = br._pools(self.m64, toks)
        c32, m32 = br._pools(self.m32, toks)
        return (m64, m32, self.range_max) if pooling == "mean" else (c64, c32, self.range_max)


def _embedder(ctx, cfg, state, pooling="mean"):
    from kaito_b200 import _native
    emb = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                           cfg["vocab_size"], cfg["max_position_embeddings"], 1, cfg["layer_norm_eps"])
    emb.set_position_offset(2)
    if pooling == "mean":
        emb.set_pooling(_native.POOL_MEAN)
    emb.load_state_dict(state)
    return emb


def _check(label, emb, ref, toks, pooling, n_sample, flat=True):
    from kaito_b200 import _native
    got = emb.embed_flat(*_native.Embedder.pack(toks)) if flat else emb.embed(toks)
    idx = br.sample([len(t) for t in toks], n_sample)
    _assert_fp64(f"mpnet {pooling} {label} ({len(toks)} seqs, {sum(len(t) for t in toks)} tok, {len(idx)} checked)", got[idx],
                 *ref([toks[i] for i in idx], pooling))
    return got


RAGGED = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 90, 91, 92, 127, 128, 129, 130, 255, 256, 257, 384, 511, 512]


def _ragged(seed, extra=21):
    g = np.random.default_rng(seed)
    lens = RAGGED + g.integers(1, 513, extra).tolist()
    return [g.integers(1000, 30000, n) for n in lens]


# ------------------------------------------------------------------------------------------------ against fp64
@pytest.mark.gpu
@pytest.mark.parametrize("pooling", ["mean", "cls"])
@pytest.mark.parametrize("regime", REGIMES)
def test_query_batch_matches_fp64(ctx, regime, pooling):
    """all-mpnet-base-v2 (mean) / multi-qa-mpnet-base (CLS) at full depth, 256 queries x 32 tokens"""
    state = _state(MPNET_BASE, regime)
    emb = _embedder(ctx, MPNET_BASE, state, pooling)
    try:
        _check(f"base {regime} 256x32", emb, Fp64MPNet(MPNET_BASE, state), _bench_queries(), pooling, 32)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_ragged_matches_fp64(ctx, pooling):
    """one batch of lengths 1..512 at full depth, stressed weights: distances in the exact (< 8), logarithmic and saturated
    (>= 91) buckets and past the +-128 clamp, across several 64-key blocks"""
    state = _state(MPNET_BASE, "stressed", seed=3)
    emb = _embedder(ctx, MPNET_BASE, state, pooling)
    ref = Fp64MPNet(MPNET_BASE, state)
    try:
        toks = _ragged(3)
        _check(f"base stressed ragged 1-512", emb, ref, toks, pooling, 10)
        long = [t for t in toks if len(t) in (91, 128, 129, 512)]
        _assert_fp64(f"mpnet {pooling} base stressed 91/128/129/512 tokens", emb.embed(long), *ref(long, pooling))
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_index_batch_matches_fp64(ctx, regime):
    """/index on a 2-layer all-mpnet-base-v2: 256 chunks x 256 tokens = 65,536 tokens through embed_flat"""
    state = _state(TWO_LAYER, regime, seed=5)
    emb = _embedder(ctx, TWO_LAYER, state)
    try:
        g = np.random.default_rng(5)
        toks = [g.integers(1000, 30000, 256) for _ in range(256)]
        _check(f"2-layer {regime} 256x256", emb, Fp64MPNet(TWO_LAYER, state), toks, "mean", 16)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_head_dim_32_matches_fp64(ctx, pooling):
    """hidden 384, 12 heads of 32 dims (the DH = 32 instantiations), ragged, stressed"""
    state = _state(HEAD32, "stressed", seed=7)
    emb = _embedder(ctx, HEAD32, state, pooling)
    try:
        _check("hidden 384 stressed ragged", emb, Fp64MPNet(HEAD32, state), _ragged(7), pooling, 12)
    finally:
        emb.destroy()


@pytest.mark.gpu
def test_zeroed_bias_is_far_off(ctx):
    """the same weights with a zero table give embeddings far past the bound: the bias is applied"""
    state = _state(TWO_LAYER, "bench", seed=9)
    toks = _ragged(9, extra=0)[:12]
    e64 = Fp64MPNet(TWO_LAYER, state)(toks, "mean")[0]
    emb = _embedder(ctx, TWO_LAYER, dict(state, **{E.MPNET_REL_BIAS: np.zeros_like(state[E.MPNET_REL_BIAS])}))
    try:
        dev = br.l2_deviation(emb.embed(toks), e64)
        print(f"zeroed bias table: L2^2 dev {dev:.2e}")
        assert dev > 1e-2, dev
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_fp16_mode_within_torch_bf16(ctx, pooling):
    """fp16 products with the bias (REL instantiations of PLANES = 1): error against fp64 at most torch bf16 autocast's"""
    import torch
    state = _state(TWO_LAYER, "bench", seed=11)
    emb = _embedder(ctx, TWO_LAYER, state, pooling)
    emb.set_precision("fp16")
    ref = Fp64MPNet(TWO_LAYER, state)
    try:
        g = np.random.default_rng(11)
        toks = [g.integers(1000, 30000, int(n)) for n in [1, 2, 17, 32, 64, 129, 300, 512] + g.integers(3, 200, 40).tolist()]
        got = emb.embed(toks)
        idx = br.sample([len(t) for t in toks], 16)
        sub = [toks[i] for i in idx]
        e64 = ref(sub, pooling)[0]
        m16 = copy.deepcopy(ref.m32).cuda()
        out = []
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            for t in sub:
                h = m16(input_ids=torch.tensor(np.asarray(t, np.int64)[None], device="cuda")).last_hidden_state[0].float()
                v = h.mean(0) if pooling == "mean" else h[0]
                out.append(torch.nn.functional.normalize(v, dim=0).double().cpu().numpy())
        e16 = np.stack(out)
        k5, t16 = float(np.abs(got[idx] - e64).max()), float(np.abs(e16 - e64).max())
        print(f"mpnet fp16 vs fp64 | {pooling} | k5 {k5:.2e} | torch bf16 {t16:.2e} | ratio {k5 / t16:.3f}")
        assert k5 <= t16, (k5, t16)
    finally:
        emb.destroy()


# ----------------------------------------------------------------------------------------------- bits and refusals
@pytest.mark.gpu
def test_cls_rows_shortcut_keeps_bits(ctx):
    """CLS pooling: the last layer on the [CLS] rows only (default) and over every token give the same bits"""
    state = _state(TWO_LAYER, "stressed", seed=13)
    emb = _embedder(ctx, TWO_LAYER, state, "cls")
    try:
        g = np.random.default_rng(13)
        toks = [g.integers(1000, 30000, int(n)) for n in g.integers(1, 300, 64)]
        short = emb.embed(toks)
        emb.debug_cls_rows(False)
        assert np.array_equal(emb.embed(toks), short)
    finally:
        emb.destroy()


@pytest.mark.gpu
def test_dev_host_and_graph_replay_keep_bits(ctx):
    """krag_embed and krag_embed_dev give the same bits, and a graph replay (third call of a shape) gives the eager bits"""
    import torch
    from kaito_b200 import _native
    state = _state(TWO_LAYER, "stressed", seed=17)
    emb = _embedder(ctx, TWO_LAYER, state)
    try:
        g = np.random.default_rng(17)
        toks = [g.integers(1000, 30000, n) for n in (3, 9, 1, 20, 130, 512)]
        toks2 = [g.integers(1000, 30000, len(t)) for t in toks]
        want = emb.embed(toks)
        assert np.array_equal(emb.embed(toks), want) and np.array_equal(emb.embed(toks), want)   # eager, capture, replay
        want2 = emb.embed(toks2)                                                                   # replay, new tokens
        assert not np.array_equal(want2, want)
        d = TWO_LAYER["hidden_size"]
        buf = torch.full((len(toks), d + 16), float("nan"), dtype=torch.float32, device="cuda")
        s = torch.cuda.Stream()
        emb.embed_dev(*_native.Embedder.pack(toks2), buf.data_ptr(), d + 16, s.cuda_stream)
        s.synchronize()
        got = buf.cpu().numpy()
        assert np.array_equal(got[:, :d], want2) and np.isnan(got[:, d:]).all()
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [31, 33])
def test_wrong_sized_bias_is_refused(ctx, rows):
    from kaito_b200 import _native
    state = _state(HEAD32, "bench", seed=19)
    state[E.MPNET_REL_BIAS] = np.zeros((rows, HEAD32["num_attention_heads"]), np.float32)
    with pytest.raises(_native.KragError) as e:
        _embedder(ctx, HEAD32, state)
    assert e.value.code == _native.KRAG_E_INVALID and E.MPNET_REL_BIAS in str(e.value), str(e.value)


# ------------------------------------------------------------------------------------------ snapshot and service
MINI = dict(HEAD32, vocab_size=len(["<s>", "<pad>", "</s>", "<unk>"] + sn.VOCAB + ["<mask>"]))


def _snapshot(tmp_path):
    from tests.test_embed_mpnet_cpu import MPNET_BASE as CFG_JSON, VOCAB, mpnet_layout
    state = _state(MINI, "bench", seed=23)
    cfg = dict(CFG_JSON, **{k: MINI[k] for k in ("num_hidden_layers", "hidden_size", "num_attention_heads", "intermediate_size",
                                                  "vocab_size")})
    mstate = {_mpnet_name(k): v for k, v in state.items() if "token_type" not in k}
    return sn.write(tmp_path / "mpnet", mpnet_layout("all-mpnet", cfg), vocab=VOCAB, state=mstate), state, VOCAB


def _texts(g, words, n, lo=3, hi=40):
    return [" ".join(g.choice(words, int(g.integers(lo, hi)))) for _ in range(n)]


@pytest.mark.gpu
def test_from_pretrained_mpnet_snapshot(ctx, tmp_path):
    """the snapshot's spec reaches the forward (mean pooling, <s> ... </s>, 384-token truncation, no query instruction); the
    embeddings are the direct MPNet embedder's, bit for bit"""
    from kaito_b200.embedding import GpuBertEmbedding
    path, state, vocab = _snapshot(tmp_path)
    words = [w for w in vocab if not w.startswith(("[", "##", "<"))]
    g = np.random.default_rng(29)
    texts = _texts(g, words, 20) + [" ".join(g.choice(words, 500))]
    ge = GpuBertEmbedding.from_pretrained(ctx, path)
    direct = _embedder(ctx, MINI, state)
    try:
        assert ge.pooling == "mean" and ge.query_instruction is None and ge.tokenizer.max_length == 384
        toks = ge.tokenizer.encode_batch(texts)
        assert len(toks[-1]) == 384 and toks[0][0] == vocab.index("<s>") and toks[0][-1] == vocab.index("</s>")
        assert np.array_equal(ge.get_text_embedding_batch(texts), direct.embed(toks))
        assert np.array_equal(ge.get_query_embedding_batch(texts[:4]), ge.get_text_embedding_batch(texts[:4]))
    finally:
        ge._emb.destroy(); direct.destroy()


@pytest.mark.gpu
def test_vector_store_retrieve_on_mpnet_snapshot(ctx, tmp_path, monkeypatch):
    """/index then /retrieve through VectorStore: every returned dense L2^2 is fp64 MPNetModel's within 1e-4, and the dense
    ranking follows fp64 wherever two fp64 distances differ by more than 1e-4"""
    from kaito_b200.embedding import GpuBertEmbedding
    from kaito_b200.vector_store import VectorStore
    monkeypatch.setenv("KRAG_COMPONENT_SCORES", "1")
    path, state, vocab = _snapshot(tmp_path)
    words = [w for w in vocab if not w.startswith(("[", "##", "<"))]
    ref = Fp64MPNet(MINI, state)
    g = np.random.default_rng(31)
    docs = [{"text": t} for t in dict.fromkeys(_texts(g, words, 60, 5, 60))]
    queries = _texts(g, words, 6, 2, 8)
    ge = GpuBertEmbedding.from_pretrained(ctx, path)
    pool = lambda texts: br.mean_pool(ref.m64, ge.tokenizer.encode_batch(texts))   # noqa: E731
    try:
        store = VectorStore(ge, ctx)
        store.index_documents("mpnet_e2e", docs)
        for q in queries:
            q64 = pool([q])[0]
            res = store.retrieve("mpnet_e2e", q, max_node_count=10)["results"]
            dense = [r for r in res if r["dense_score"] is not None]
            assert dense, q
            l2 = ((pool([r["text"] for r in dense]) - q64) ** 2).sum(1)
            assert np.abs(np.array([r["dense_score"] for r in dense]) - l2).max() < 1e-4, q
            ranked = store.dense_candidates("mpnet_e2e", q, len(docs))
            assert len(ranked) == len(docs)
            r64 = ((pool([n.text for n, _ in ranked]) - q64) ** 2).sum(1)
            assert np.abs(np.array([s for _, s in ranked]) - r64).max() < 1e-4, q
            assert (np.diff(r64) > -1e-4).all(), (q, np.diff(r64).min())
    finally:
        ge._emb.destroy()
