"""K5 as a nomic-embed-text encoder (nomic_bert): rotary positions applied to Q and K in the QKV GEMM epilogue
(gemm_f16s_kernel / splitk_reduce_kernel EP_ROPE), the SwiGLU FFN1 epilogue (EP_SWIGLU), no position table, no biases.
Held to the bounds of tests/test_gpu_embed.py against transformers.NomicBertModel in fp64, mean-pooled and normalised in
numpy: the L2^2 score against 64 unit rows moves by less than 1e-4 and the error is at most F = 40 times torch fp32's own.
Two weight regimes: "bench" = bert_reference.random_state's magnitudes with an extra gate matrix (full depth); "stressed" =
outlier LayerNorm channels (gamma 10-20) and query / key weights scaled so that each layer's attention scores have a std of
~12 (2 layers: see STRESS_DEPTH).
Also: every linear_plan choice on the rotary QKV and the gated FFN1, sequences of 8192 tokens (positions past nomic's 2048
trained ones run plain RoPE), the CLS-rows shortcut, device / host output and graph replay give the same bits; rotary off
or the gate left out move the embeddings far past the bound; wrong-sized or missing gate tensors and a missing position
table are refused at finalize; fp16 mode stays within torch bf16 autocast's error; a hub-format snapshot goes through
GpuBertEmbedding.from_pretrained and a VectorStore /retrieve."""
import copy

import numpy as np
import pytest

from kaito_b200 import embedding as E
from tests import bert_reference as br
from tests import st_snapshot as sn
from tests.test_embed_nomic_cpu import native_state, nomic_layout, NOMIC_HUB
from tests.test_gpu_embed import _assert_fp64, _bench_queries

NOMIC_BASE = dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=30528,
                  max_position_embeddings=8192, type_vocab_size=2, layer_norm_eps=1e-12, rotary_base=1000.0)   # v1 / v1.5
TWO_LAYER = dict(NOMIC_BASE, num_hidden_layers=2)
HEAD32 = dict(NOMIC_BASE, num_hidden_layers=2, hidden_size=384, intermediate_size=1536)   # 12 heads of 32 dims
SMALL_INTER = dict(HEAD32, intermediate_size=512)
REGIMES = ["bench", "stressed"]
# Stressed weights run on 2 layers.  Random nomic weights (no biases, a gated FFN) amplify a perturbation layer after layer:
# at 12 layers torch fp32 itself is 1e-3 .. 2e-1 (L2^2) from fp64 under this stress, so no fp32 forward can meet the 1e-4
# contract there (K5 measured 2.0 - 3.7x torch fp32's error on those batches; H100 SXM).  Bench weights run at full depth.
STRESS_DEPTH = 2
SMS, WS_FLOATS = 132, 4 << 20            # H100 SXM; Embedder::WS_FLOATS


def _nomic_torch_config(cfg):
    from transformers import NomicBertConfig
    kw = {k: v for k, v in cfg.items() if k != "rotary_base"}
    return NomicBertConfig(**kw, hidden_act="silu", rope_parameters={"rope_type": "default", "rope_theta": cfg["rotary_base"]},
                           attn_implementation="eager")


def _hub_state(cfg, seed):
    """hub-named weights with random_state's magnitudes: embeddings N(0, 0.02), matrices N(0, 0.06), LayerNorm gamma N(1, 0.1)"""
    g = np.random.default_rng(seed)
    d, i = cfg["hidden_size"], cfg["intermediate_size"]
    n = lambda std, *s, mean=0.0: (mean + std * g.standard_normal(s, dtype=np.float32)).astype(np.float32)   # noqa: E731
    st = {"embeddings.word_embeddings.weight": n(0.02, cfg["vocab_size"], d), "embeddings.token_type_embeddings.weight": n(0.02, 2, d),
          "emb_ln.weight": n(0.1, d, mean=1.0), "emb_ln.bias": n(0.05, d)}
    for l in range(cfg["num_hidden_layers"]):
        p = f"encoder.layers.{l}."
        st.update({p + "attn.Wqkv.weight": n(0.06, 3 * d, d), p + "attn.out_proj.weight": n(0.06, d, d),
                   p + "mlp.fc11.weight": n(0.06, i, d), p + "mlp.fc12.weight": n(0.06, i, d), p + "mlp.fc2.weight": n(0.06, d, i)})
        for ln in ("norm1", "norm2"):
            st[p + ln + ".weight"], st[p + ln + ".bias"] = n(0.1, d, mean=1.0), n(0.05, d)
    return st


class Fp64Nomic:
    """transformers.NomicBertModel (eager attention) in fp64 and its fp32 twin, with Linear range hooks"""

    def __init__(self, cfg, hub, device="cpu"):
        import torch
        from transformers import NomicBertModel
        from transformers.initialization import no_init_weights
        with no_init_weights():
            self.m64 = NomicBertModel(_nomic_torch_config(cfg)).double().eval()
        sd = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in native_state(hub).items()}
        missing, unexpected = self.m64.load_state_dict(sd, strict=False)
        assert not unexpected and not [k for k in missing if not k.endswith(("position_ids", "token_type_ids"))], missing
        self.m32 = copy.deepcopy(self.m64).float()
        self.m64.to(device); self.m32.to(device)
        self.device, self.range_max = device, 0.0
        for mod in self.m64.modules():
            if isinstance(mod, torch.nn.Linear):
                mod.register_forward_hook(lambda m, i, o: setattr(self, "range_max", max(self.range_max, float(i[0].abs().max()),
                                                                                        float(o.abs().max()))))

    def _pools(self, m, toks):
        import torch
        cls, mean = [], []
        with torch.no_grad():
            for t in toks:
                h = m(input_ids=torch.tensor(np.asarray(t, np.int64)[None], device=self.device)).last_hidden_state[0]
                for out, v in ((cls, h[0]), (mean, h.mean(0))):
                    out.append((v / torch.clamp(torch.linalg.norm(v), min=1e-12)).double().cpu().numpy())
        return np.stack(cls), np.stack(mean)

    def __call__(self, toks, pooling="mean"):
        """(fp64 embeddings, fp32 embeddings, largest Linear operand of the fp64 forward) of each sequence run alone"""
        self.range_max = 0.0
        c64, m64 = self._pools(self.m64, toks)
        c32, m32 = self._pools(self.m32, toks)
        return (m64, m32, self.range_max) if pooling == "mean" else (c64, c32, self.range_max)


def _state(cfg, regime, seed=0):
    """(hub-named weights, their Fp64Nomic)"""
    import torch
    st = _hub_state(cfg, seed)
    if regime == "bench":
        return st, Fp64Nomic(cfg, st)
    assert cfg["num_hidden_layers"] <= STRESS_DEPTH, "stressed nomic weights are ill-conditioned past STRESS_DEPTH layers"
    g = np.random.default_rng(seed + 1000)
    ch = g.choice(cfg["hidden_size"], 3, replace=False)
    for k in [k for k in st if k.endswith(("emb_ln.weight", "norm1.weight", "norm2.weight"))]:
        st[k][ch] = g.uniform(10.0, 20.0, 3).astype(np.float32)
    ref = Fp64Nomic(cfg, st)
    calib = [g.integers(1000, 30000, 48) for _ in range(2)]
    d, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    for l in range(cfg["num_hidden_layers"]):       # scale Wq, Wk of layer l so that its scores have std ~12
        att, got, scores = ref.m64.layers[l].self_attn, {}, []
        hooks = [getattr(att, n).register_forward_hook(lambda m, i, o, n=n: got.__setitem__(n, o)) for n in ("q_proj", "k_proj")]
        with torch.no_grad():
            for t in calib:
                ref.m64(input_ids=torch.tensor(np.asarray(t, np.int64)[None]))
                q, k = (got[n][0].view(len(t), heads, -1).transpose(0, 1) for n in ("q_proj", "k_proj"))
                scores.append((q @ k.transpose(1, 2) / np.sqrt(d // heads)).flatten())
        for h in hooks:
            h.remove()
        c = np.sqrt(12.0 / float(torch.cat(scores).std()))
        key = f"encoder.layers.{l}.attn.Wqkv.weight"
        st[key][:2 * d] *= np.float32(c)
        with torch.no_grad():
            for n, rows in (("q_proj", slice(0, d)), ("k_proj", slice(d, 2 * d))):
                getattr(att, n).weight.copy_(torch.from_numpy(st[key][rows].astype(np.float64)))
    ref.m32 = copy.deepcopy(ref.m64).float()
    return st, ref


def _embedder(ctx, cfg, hub, pooling="mean", rotary=True, state=None):
    from kaito_b200 import _native
    st = state if state is not None else E.nomic_state(hub, cfg)
    emb = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                           cfg["vocab_size"], cfg["max_position_embeddings"], st["embeddings.token_type_embeddings.weight"].shape[0],
                           cfg["layer_norm_eps"])
    try:
        if pooling == "mean":
            emb.set_pooling(_native.POOL_MEAN)
        if rotary:
            emb.set_rotary(cfg["rotary_base"])
        emb.load_state_dict(st)
    except Exception:
        emb.destroy()
        raise
    return emb


def _check(label, emb, ref, toks, pooling, n_sample, flat=True):
    from kaito_b200 import _native
    got = emb.embed_flat(*_native.Embedder.pack(toks)) if flat else emb.embed(toks)
    idx = br.sample([len(t) for t in toks], n_sample)
    _assert_fp64(f"nomic {pooling} {label} ({len(toks)} seqs, {sum(len(t) for t in toks)} tok, {len(idx)} checked)", got[idx],
                 *ref([toks[i] for i in idx], pooling))
    return got


RAGGED = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 130, 255, 256, 257, 384, 511, 512]


def _ragged(seed, extra=21):
    g = np.random.default_rng(seed)
    return [g.integers(1000, 30000, n) for n in RAGGED + g.integers(1, 513, extra).tolist()]


# ------------------------------------------------------------------------------------------------ against fp64
@pytest.mark.gpu
@pytest.mark.parametrize("regime,cfg", [("bench", NOMIC_BASE), ("stressed", TWO_LAYER)], ids=["bench-12-layers", "stressed-2-layers"])
def test_query_batch_matches_fp64(ctx, regime, cfg):
    """nomic-embed-text-v1.5's shape (768, 12 heads, 3072), 256 queries x 32 tokens, mean pooling: bench weights at full
    depth, stressed weights on 2 layers (see STRESS_DEPTH)"""
    hub, ref = _state(cfg, regime)
    emb = _embedder(ctx, cfg, hub)
    try:
        _check(f"{cfg['num_hidden_layers']}-layer {regime} 256x32", emb, ref, _bench_queries(), "mean", 32)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_ragged_matches_fp64(ctx, pooling):
    """one batch of lengths 1..512 on 2 layers, stressed weights"""
    hub, ref = _state(TWO_LAYER, "stressed", seed=3)
    emb = _embedder(ctx, TWO_LAYER, hub, pooling)
    try:
        _check("2-layer stressed ragged 1-512", emb, ref, _ragged(3), pooling, 10)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_index_batch_matches_fp64(ctx, regime):
    """/index on a 2-layer nomic: 256 chunks x 256 tokens = 65,536 tokens through embed_flat"""
    hub, ref = _state(TWO_LAYER, regime, seed=5)
    emb = _embedder(ctx, TWO_LAYER, hub)
    try:
        g = np.random.default_rng(5)
        _check(f"2-layer {regime} 256x256", emb, ref, [g.integers(1000, 30000, 256) for _ in range(256)], "mean", 16)
    finally:
        emb.destroy()


@pytest.mark.gpu
def test_long_sequences_match_fp64(ctx):
    """sequences up to 8192 tokens (2 layers, stressed): positions past the 2048 trained ones, angles up to 8191 rad"""
    hub, ref = _state(TWO_LAYER, "stressed", seed=7)
    ref = Fp64Nomic(TWO_LAYER, hub, device="cuda")          # the fp64 attention matrix of 8192 tokens is 6.4 GB
    emb = _embedder(ctx, TWO_LAYER, hub)
    try:
        g = np.random.default_rng(7)
        toks = [g.integers(1000, 30000, n) for n in (8192, 3000, 2049, 5)]
        _check("2-layer stressed to 8192 tokens", emb, ref, toks, "mean", 4)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_head_dim_32_matches_fp64(ctx, pooling):
    """hidden 384, 12 heads of 32 dims, ragged, stressed"""
    hub, ref = _state(HEAD32, "stressed", seed=9)
    emb = _embedder(ctx, HEAD32, hub, pooling)
    try:
        _check("hidden 384 stressed ragged", emb, ref, _ragged(9), pooling, 12)
    finally:
        emb.destroy()


def linear_plan(M, N, K):
    """embed.cu linear_plan's (tile width, K splits) for a split-fp16 layer without LayerNorm, workspace present"""
    m_tiles = -(-M // 128)
    if m_tiles * (N // 128) < SMS // 2 and N % 64 == 0 and K % 64 == 0:
        bn = 32 if m_tiles == 1 else (128 if K >= 2048 and N % 128 == 0 else 64)
        ctas, kb = m_tiles * (N // bn), K // 64
        if ctas <= SMS // 3:
            for sp in range(min(SMS // ctas, 8), 1, -1):
                if kb % sp == 0 and kb // sp >= 2 and sp * M * N <= WS_FLOATS:
                    return bn, sp
        return bn, 1
    return 128, 1


# (label, config, token counts, (QKV plan, FFN1 plan) the rule gives)
PLANS = [
    ("128x32 one query", TWO_LAYER, [32], ((32, 1), (32, 1))),           # a 64-dim head spans two 32-column tiles
    ("128x64", TWO_LAYER, [100, 100], ((64, 1), (128, 1))),
    ("128x128", TWO_LAYER, [512, 512], ((128, 1), (128, 1))),
    ("split-K", SMALL_INTER, [32], ((32, 3), (32, 3))),                  # N = 1152: 36 CTAs; N = 2 * 512: 32 CTAs
    ("split-K 128x64", SMALL_INTER, [100, 100], ((64, 3), (64, 3))),
]


@pytest.mark.gpu
@pytest.mark.parametrize("label,cfg,lens,plans", PLANS, ids=[p[0] for p in PLANS])
def test_every_plan_matches_fp64(ctx, label, cfg, lens, plans):
    """the rotary QKV epilogue and the gated FFN1 epilogue under each tile width and the split-K reduce"""
    d, n_tok = cfg["hidden_size"], sum(lens)
    assert (linear_plan(n_tok, 3 * d, d), linear_plan(n_tok, 2 * cfg["intermediate_size"], d)) == plans
    hub, ref = _state(cfg, "stressed", seed=11)
    emb = _embedder(ctx, cfg, hub)
    try:
        g = np.random.default_rng(11)
        _check(label, emb, ref, [g.integers(1000, 30000, n) for n in lens], "mean", 4, flat=False)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_fp16_mode_within_torch_bf16(ctx, pooling):
    """fp16 products (PLANES = 1 instantiations, 128 x 256 tiles at 2,048+ tokens): error against fp64 at most torch bf16
    autocast's"""
    import torch
    hub, ref = _state(TWO_LAYER, "bench", seed=13)
    emb = _embedder(ctx, TWO_LAYER, hub, pooling)
    emb.set_precision("fp16")
    try:
        g = np.random.default_rng(13)
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
        k5, t16 = float(np.abs(got[idx] - e64).max()), float(np.abs(np.stack(out) - e64).max())
        print(f"nomic fp16 vs fp64 | {pooling} | k5 {k5:.2e} | torch bf16 {t16:.2e} | ratio {k5 / t16:.3f}")
        assert k5 <= t16, (k5, t16)
    finally:
        emb.destroy()


# ----------------------------------------------------------------------------------------------- bits and sensitivity
@pytest.mark.gpu
def test_cls_rows_shortcut_keeps_bits(ctx):
    """CLS pooling with the gated FFN: the last layer on the [CLS] rows only (default) and over every token give the same bits"""
    hub, _ = _state(TWO_LAYER, "bench", seed=15)
    emb = _embedder(ctx, TWO_LAYER, hub, "cls")
    try:
        g = np.random.default_rng(15)
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
    hub, _ = _state(TWO_LAYER, "bench", seed=17)
    emb = _embedder(ctx, TWO_LAYER, hub)
    try:
        g = np.random.default_rng(17)
        toks = [g.integers(1000, 30000, n) for n in (3, 9, 1, 20, 130, 512)]
        toks2 = [g.integers(1000, 30000, len(t)) for t in toks]
        want = emb.embed(toks)
        assert np.array_equal(emb.embed(toks), want) and np.array_equal(emb.embed(toks), want)   # eager, capture, replay
        want2 = emb.embed(toks2)
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
@pytest.mark.parametrize("change", ["rotary off", "no gate"])
def test_each_piece_moves_the_embeddings(ctx, change):
    """rotary off (a zero position table instead) or the gate left out (GELU on the up projection) put the embeddings far
    past the bound: both epilogues are exercised"""
    hub, ref = _state(TWO_LAYER, "bench", seed=19)
    g = np.random.default_rng(19)
    toks = [g.integers(1000, 30000, int(n)) for n in (5, 40, 129, 300)]
    st = E.nomic_state(hub, TWO_LAYER)
    if change == "rotary off":
        st["embeddings.position_embeddings.weight"] = np.zeros((TWO_LAYER["max_position_embeddings"], TWO_LAYER["hidden_size"]), np.float32)
    else:
        st = {k: v for k, v in st.items() if ".intermediate.gate." not in k}
    emb = _embedder(ctx, TWO_LAYER, hub, rotary=change != "rotary off", state=st)
    try:
        dev = br.l2_deviation(emb.embed(toks), ref(toks)[0])
        print(f"nomic {change}: L2^2 dev {dev:.2e}")
        assert dev > 1e-2, dev
    finally:
        emb.destroy()


REFUSED = [
    ("gate 1 row short", lambda st: st.__setitem__("encoder.layer.1.intermediate.gate.weight",
                                                   st["encoder.layer.1.intermediate.gate.weight"][:-1]),
     "encoder.layer.1.intermediate.gate.weight", True),
    ("gate missing on layer 1", lambda st: st.pop("encoder.layer.1.intermediate.gate.weight"),
     "encoder.layer.1.intermediate.gate.weight", True),
    ("gate bias missing", lambda st: st.pop("encoder.layer.0.intermediate.gate.bias"), "encoder.layer.0.intermediate.gate.bias", True),
    ("no position table, rotary off", lambda st: None, "embeddings.position_embeddings.weight", False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("label,edit,name,rotary", REFUSED, ids=[r[0] for r in REFUSED])
def test_finalize_refusals_name_the_tensor(ctx, label, edit, name, rotary):
    from kaito_b200 import _native
    hub = _hub_state(HEAD32, 21)
    st = E.nomic_state(hub, HEAD32)
    edit(st)
    with pytest.raises(_native.KragError) as e:
        _embedder(ctx, HEAD32, hub, rotary=rotary, state=st)
    assert e.value.code == _native.KRAG_E_INVALID and name in str(e.value), str(e.value)


# ------------------------------------------------------------------------------------------ snapshot and service
MINI = dict(HEAD32, vocab_size=len(sn.VOCAB), max_position_embeddings=2048)


def _snapshot(tmp_path):
    hub, ref = _state(MINI, "bench", seed=23)
    cfg = dict(NOMIC_HUB, n_layer=MINI["num_hidden_layers"], n_embd=MINI["hidden_size"], n_head=MINI["num_attention_heads"],
               n_inner=MINI["intermediate_size"], vocab_size=MINI["vocab_size"], n_positions=MINI["max_position_embeddings"])
    return sn.write(tmp_path / "nomic", nomic_layout(cfg, max_seq_length=2048), vocab=sn.VOCAB, state=hub), hub, ref


def _texts(g, words, n, lo=3, hi=40):
    return [" ".join(g.choice(words, int(g.integers(lo, hi)))) for _ in range(n)]


@pytest.mark.gpu
def test_from_pretrained_nomic_snapshot(ctx, tmp_path):
    """the hub snapshot's spec reaches the forward: mean pooling, the task prefixes, rotary + gated; the embeddings are the
    direct embedder's bit for bit and fp64 NomicBertModel's within the bound"""
    from kaito_b200.embedding import GpuBertEmbedding
    path, hub, ref = _snapshot(tmp_path)
    words = [w for w in sn.VOCAB if not w.startswith(("[", "##"))]
    g = np.random.default_rng(29)
    texts = _texts(g, words, 20)
    ge = GpuBertEmbedding.from_pretrained(ctx, path)
    direct = _embedder(ctx, MINI, hub)
    try:
        assert ge.pooling == "mean" and ge.query_instruction == "search_query: " and ge.text_instruction == "search_document: "
        docs = ge.tokenizer.encode_batch(["search_document: " + t for t in texts])
        got = ge.get_text_embedding_batch(texts)
        assert np.array_equal(got, direct.embed(docs))
        _assert_fp64("nomic snapshot documents", got, *ref(docs))
        qs = ge.tokenizer.encode_batch(["search_query: " + t for t in texts[:4]])
        assert np.array_equal(ge.get_query_embedding_batch(texts[:4]), direct.embed(qs))
    finally:
        ge._emb.destroy(); direct.destroy()


@pytest.mark.gpu
def test_vector_store_retrieve_on_nomic_snapshot(ctx, tmp_path, monkeypatch):
    """/index then /retrieve through VectorStore: every returned dense L2^2 is fp64 NomicBertModel's within 1e-4 (documents
    behind "search_document: ", the query behind "search_query: ")"""
    from kaito_b200.embedding import GpuBertEmbedding
    from kaito_b200.vector_store import VectorStore
    monkeypatch.setenv("KRAG_COMPONENT_SCORES", "1")
    path, hub, ref = _snapshot(tmp_path)
    words = [w for w in sn.VOCAB if not w.startswith(("[", "##"))]
    g = np.random.default_rng(31)
    docs = [{"text": t} for t in dict.fromkeys(_texts(g, words, 60, 5, 60))]
    queries = _texts(g, words, 4, 2, 8)
    ge = GpuBertEmbedding.from_pretrained(ctx, path)
    pool = lambda texts, prefix: ref([np.asarray(t) for t in ge.tokenizer.encode_batch([prefix + x for x in texts])])[0]   # noqa: E731
    try:
        store = VectorStore(ge, ctx)
        store.index_documents("nomic_e2e", docs)
        for q in queries:
            q64 = pool([q], "search_query: ")[0]
            res = store.retrieve("nomic_e2e", q, max_node_count=10)["results"]
            dense = [r for r in res if r["dense_score"] is not None]
            assert dense, q
            l2 = ((pool([r["text"] for r in dense], "search_document: ") - q64) ** 2).sum(1)
            assert np.abs(np.array([r["dense_score"] for r in dense]) - l2).max() < 1e-4, q
    finally:
        ge._emb.destroy()
