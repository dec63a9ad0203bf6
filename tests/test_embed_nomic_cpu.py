"""nomic-embed-text v1 / v1.5 (nomic_bert) without a GPU: read_snapshot_spec on snapshots laid out with the hub's
custom-code config and with transformers' NomicBertConfig, its refusals (each naming its file and field), the two tensor
name sets mapped onto the same K5 tensors, the rotary cos / sin K5 applies against transformers' NomicBertRotaryEmbedding,
and the task prefixes on documents and on both query paths."""
import numpy as np
import pytest

from kaito_b200 import embedding as E
from kaito_b200.embedding import read_snapshot_spec
from tests import st_snapshot as sn

# config.json of nomic-ai/nomic-embed-text-v1.5 under the hub's custom-code names (restated: no snapshot offline)
NOMIC_HUB = dict(activation_function="swiglu", architectures=["NomicBertModel"], attn_pdrop=0.0, bos_token_id=None,
                 causal=False, dense_seq_output=True, embd_pdrop=0.0, eos_token_id=None, fused_bias_fc=True,
                 fused_dropout_add_ln=True, initializer_range=0.02, layer_norm_epsilon=1e-12, max_trained_positions=2048,
                 mlp_fc1_bias=False, mlp_fc2_bias=False, model_type="nomic_bert", n_embd=768, n_head=12, n_inner=3072,
                 n_layer=12, n_positions=8192, pad_vocab_size_multiple=64, parallel_block=False, parallel_block_tied_norm=False,
                 prenorm=False, qkv_proj_bias=False, reorder_and_upcast_attn=False, resid_pdrop=0.0, rotary_emb_base=1000,
                 rotary_emb_fraction=1.0, rotary_emb_interleaved=False, rotary_emb_scale_base=None, rotary_scaling_factor=None,
                 scale_attn_by_inverse_layer_idx=False, scale_attn_weights=True, summary_activation=None,
                 summary_first_dropout=0.0, summary_proj_to_labels=True, summary_type="cls_index", summary_use_proj=True,
                 type_vocab_size=2, use_cache=True, use_flash_attn=True, use_rms_norm=False, use_xentropy=True, vocab_size=30528)
# the same model under transformers' NomicBertConfig names
NOMIC_NATIVE = dict(architectures=["NomicBertModel"], hidden_act="silu", hidden_size=768, intermediate_size=3072,
                    layer_norm_eps=1e-12, max_position_embeddings=8192, model_type="nomic_bert", num_attention_heads=12,
                    num_hidden_layers=12, rope_parameters={"rope_type": "default", "rope_theta": 1000.0}, type_vocab_size=2,
                    vocab_size=30528)
K5_CONFIG = dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072,
                 max_position_embeddings=8192, vocab_size=30528, type_vocab_size=2, layer_norm_eps=1e-12, rotary_base=1000.0)


def nomic_layout(config=None, max_seq_length=8192):
    """{file name: JSON content} of a nomic-embed-text-v1.5 snapshot: Transformer, mean Pooling, Normalize, 8192 tokens,
    the bert-base-uncased tokenizer"""
    cfg = dict(config or NOMIC_HUB)
    d = cfg.get("n_embd", cfg.get("hidden_size"))
    return {
        "config.json": cfg,
        "tokenizer_config.json": {"cls_token": "[CLS]", "do_lower_case": True, "mask_token": "[MASK]", "model_max_length": 8192,
                                  "pad_token": "[PAD]", "sep_token": "[SEP]", "strip_accents": None,
                                  "tokenize_chinese_chars": True, "tokenizer_class": "BertTokenizer", "unk_token": "[UNK]"},
        "sentence_bert_config.json": {"max_seq_length": max_seq_length, "do_lower_case": False},
        "modules.json": [{"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
                         {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
                         {"idx": 2, "name": "2", "path": "2_Normalize", "type": "sentence_transformers.models.Normalize"}],
        "1_Pooling/config.json": sn.pooling_config(d, "mean_tokens"),
    }


def _write(tmp_path, files, name="snap"):
    return sn.write(tmp_path / name, files, vocab=sn.VOCAB)


# ------------------------------------------------------------------------------------------------ snapshot spec
@pytest.mark.parametrize("form", ["hub", "native"])
def test_nomic_layout(tmp_path, form):
    spec = read_snapshot_spec(_write(tmp_path, nomic_layout(NOMIC_HUB if form == "hub" else NOMIC_NATIVE)))
    assert spec == {"pooling": "mean", "max_length": 8192, "do_lower_case": True, "query_instruction": "search_query: ",
                    "text_instruction": "search_document: ", "model_type": "nomic_bert", "config": K5_CONFIG}


def test_max_length_from_n_positions(tmp_path):
    """no sentence_bert_config.json: min(model_max_length, n_positions)"""
    files = nomic_layout(dict(NOMIC_HUB, n_positions=2048))
    files["sentence_bert_config.json"] = None
    assert read_snapshot_spec(_write(tmp_path, files))["max_length"] == 2048


def test_existing_specs_are_unchanged(tmp_path):
    """BERT and MPNet specs have no nomic keys"""
    from tests.test_embed_mpnet_cpu import VOCAB, mpnet_layout
    assert set(read_snapshot_spec(_write(tmp_path, sn.layout("minilm"), "bert"))) == \
        {"pooling", "max_length", "do_lower_case", "query_instruction"}
    mp = read_snapshot_spec(sn.write(tmp_path / "mpnet", mpnet_layout(), vocab=VOCAB))
    assert "text_instruction" not in mp and mp["query_instruction"] is None and mp["model_type"] == "mpnet"


def _without(cfg, field):
    return {k: v for k, v in cfg.items() if k != field}


REFUSALS = [
    ("interleaved", dict(NOMIC_HUB, rotary_emb_interleaved=True), "rotary_emb_interleaved"),
    ("fraction 0.5", dict(NOMIC_HUB, rotary_emb_fraction=0.5), "rotary_emb_fraction"),
    ("fraction absent", _without(NOMIC_HUB, "rotary_emb_fraction"), "rotary_emb_fraction"),
    ("dynamic NTK", dict(NOMIC_HUB, rotary_scaling_factor=2.0), "rotary_scaling_factor"),
    ("prenorm", dict(NOMIC_HUB, prenorm=True), "prenorm"),
    ("rms norm", dict(NOMIC_HUB, use_rms_norm=True), "use_rms_norm"),
    ("causal", dict(NOMIC_HUB, causal=True), "causal"),
    ("qkv bias", dict(NOMIC_HUB, qkv_proj_bias=True), "qkv_proj_bias"),
    ("fc1 bias", dict(NOMIC_HUB, mlp_fc1_bias=True), "mlp_fc1_bias"),
    ("fc2 bias", dict(NOMIC_HUB, mlp_fc2_bias=True), "mlp_fc2_bias"),
    ("gelu", dict(NOMIC_HUB, activation_function="gelu"), "activation_function"),
    ("base absent", _without(NOMIC_HUB, "rotary_emb_base"), "rotary_emb_base"),
    ("head dim 48", dict(NOMIC_HUB, n_head=16), "n_head"),
    ("inner 3000", dict(NOMIC_HUB, n_inner=3000), "n_inner"),
    ("hidden 1152", dict(NOMIC_HUB, n_embd=1152, n_head=18), "n_embd"),
    ("native gelu", dict(NOMIC_NATIVE, hidden_act="gelu"), "hidden_act"),
    ("native dynamic rope", dict(NOMIC_NATIVE, rope_parameters={"rope_type": "dynamic", "rope_theta": 1000.0, "factor": 2.0}),
     "rope_type"),
    ("native head 48", dict(NOMIC_NATIVE, num_attention_heads=16), "num_attention_heads"),
]


@pytest.mark.parametrize("label,cfg,field", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_nomic_refusals_name_file_and_field(tmp_path, label, cfg, field):
    with pytest.raises(ValueError) as e:
        read_snapshot_spec(_write(tmp_path, nomic_layout(cfg)))
    assert "config.json" in str(e.value) and field in str(e.value), str(e.value)


def test_max_seq_length_past_n_positions_is_refused(tmp_path):
    with pytest.raises(ValueError) as e:
        read_snapshot_spec(_write(tmp_path, nomic_layout(max_seq_length=8193)))
    assert "sentence_bert_config.json" in str(e.value) and "n_positions 8192" in str(e.value), str(e.value)


# ------------------------------------------------------------------------------------------------ tensor names
SMALL = dict(num_hidden_layers=2, hidden_size=128, num_attention_heads=2, intermediate_size=256, vocab_size=64,
             max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12, rotary_base=1000.0)


def hub_state(cfg, seed=0):
    """a nomic checkpoint under the hub's names (Wqkv rows [q; k; v], fc11 = up, fc12 = gate), no biases"""
    g = np.random.default_rng(seed)
    d, i = cfg["hidden_size"], cfg["intermediate_size"]
    n = lambda *s: g.standard_normal(s).astype(np.float32)   # noqa: E731
    st = {"embeddings.word_embeddings.weight": n(cfg["vocab_size"], d), "embeddings.token_type_embeddings.weight": n(2, d),
          "emb_ln.weight": n(d), "emb_ln.bias": n(d)}
    for l in range(cfg["num_hidden_layers"]):
        p = f"encoder.layers.{l}."
        st.update({p + "attn.Wqkv.weight": n(3 * d, d), p + "attn.out_proj.weight": n(d, d), p + "mlp.fc11.weight": n(i, d),
                   p + "mlp.fc12.weight": n(i, d), p + "mlp.fc2.weight": n(d, i), p + "norm1.weight": n(d), p + "norm1.bias": n(d),
                   p + "norm2.weight": n(d), p + "norm2.bias": n(d)})
    return st


def native_state(hub):
    """the same weights under transformers' NomicBertModel names (its conversion mapping, Wqkv chunked along dim 0)"""
    import torch
    out = {"embeddings.word_embeddings.weight": hub["embeddings.word_embeddings.weight"],
           "embeddings.token_type_embeddings.weight": hub["embeddings.token_type_embeddings.weight"],
           "embeddings.LayerNorm.weight": hub["emb_ln.weight"], "embeddings.LayerNorm.bias": hub["emb_ln.bias"]}
    l = 0
    while f"encoder.layers.{l}.attn.Wqkv.weight" in hub:
        h, p = f"encoder.layers.{l}.", f"layers.{l}."
        q, k, v = torch.chunk(torch.from_numpy(hub[h + "attn.Wqkv.weight"]), 3, dim=0)
        out.update({p + "self_attn.q_proj.weight": q.numpy(), p + "self_attn.k_proj.weight": k.numpy(),
                    p + "self_attn.v_proj.weight": v.numpy(), p + "self_attn.o_proj.weight": hub[h + "attn.out_proj.weight"],
                    p + "mlp.up_proj.weight": hub[h + "mlp.fc11.weight"], p + "mlp.gate_proj.weight": hub[h + "mlp.fc12.weight"],
                    p + "mlp.down_proj.weight": hub[h + "mlp.fc2.weight"],
                    p + "post_attention_layernorm.weight": hub[h + "norm1.weight"], p + "post_attention_layernorm.bias": hub[h + "norm1.bias"],
                    p + "post_mlp_layernorm.weight": hub[h + "norm2.weight"], p + "post_mlp_layernorm.bias": hub[h + "norm2.bias"]})
        l += 1
    return out


def _k5_names(cfg):
    names = {"embeddings.word_embeddings.weight", "embeddings.token_type_embeddings.weight", "embeddings.LayerNorm.weight",
             "embeddings.LayerNorm.bias"}
    for l in range(cfg["num_hidden_layers"]):
        for nm in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense",
                   "intermediate.dense", "intermediate.gate", "output.dense", "attention.output.LayerNorm", "output.LayerNorm"):
            names |= {f"encoder.layer.{l}.{nm}.weight", f"encoder.layer.{l}.{nm}.bias"}
    return names


def test_both_name_sets_map_onto_the_same_k5_tensors():
    hub = hub_state(SMALL)
    a, b = E.nomic_state(hub, SMALL), E.nomic_state(native_state(hub), SMALL)
    assert set(a) == set(b) == _k5_names(SMALL)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    d = SMALL["hidden_size"]
    w = hub["encoder.layers.1.attn.Wqkv.weight"]
    assert np.array_equal(a["encoder.layer.1.attention.self.key.weight"], w[d:2 * d])
    assert np.array_equal(a["encoder.layer.1.intermediate.gate.weight"], hub["encoder.layers.1.mlp.fc12.weight"])
    assert np.array_equal(a["encoder.layer.1.intermediate.dense.weight"], hub["encoder.layers.1.mlp.fc11.weight"])
    assert not a["encoder.layer.0.attention.self.query.bias"].any() and a["encoder.layer.0.intermediate.gate.bias"].shape == (256,)


def test_native_names_load_into_transformers():
    """the native name set is NomicBertModel's own: it loads with nothing missing or unexpected"""
    import torch
    from transformers import NomicBertConfig, NomicBertModel
    from transformers.initialization import no_init_weights
    cfg = {k: v for k, v in SMALL.items() if k != "rotary_base"}
    with no_init_weights():
        m = NomicBertModel(NomicBertConfig(**cfg, hidden_act="silu", rope_parameters={"rope_type": "default", "rope_theta": 1000.0}))
    sd = {k: torch.from_numpy(v) for k, v in native_state(hub_state(SMALL)).items()}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and not [k for k in missing if not k.endswith(("position_ids", "token_type_ids"))], (missing, unexpected)


def test_no_token_type_table_gets_a_zero_row():
    hub = hub_state(SMALL)
    del hub["embeddings.token_type_embeddings.weight"]
    st = E.nomic_state(hub, SMALL)
    assert st["embeddings.token_type_embeddings.weight"].shape == (1, 128) and not st["embeddings.token_type_embeddings.weight"].any()


# ------------------------------------------------------------------------------------------------ rotary angles
@pytest.mark.parametrize("dh", [64, 32])
def test_rotary_cos_sin_match_transformers(dh):
    """the cos / sin of the table K5 builds are within 1 ulp of NomicBertRotaryEmbedding's at every position in [0, 8192)"""
    import torch
    from transformers import NomicBertConfig
    from transformers.models.nomic_bert.modeling_nomic_bert import NomicBertRotaryEmbedding
    from kaito_b200 import _native
    cfg = NomicBertConfig(hidden_size=4 * dh, num_attention_heads=4, max_position_embeddings=8192,
                          rope_parameters={"rope_type": "default", "rope_theta": 1000.0})
    rot = NomicBertRotaryEmbedding(cfg)
    pos = torch.arange(8192)[None]
    cos, sin = rot(torch.zeros(1, 8192, dh), pos)
    want_c, want_s = cos[0, :, :dh // 2].numpy(), sin[0, :, :dh // 2].numpy()
    assert np.array_equal(cos[0, :, :dh // 2], cos[0, :, dh // 2:])      # the two halves of a head share the angle
    got = [_native.debug_rotary_cos_sin(1000.0, dh, p) for p in range(8192)]
    got_c, got_s = np.stack([g[0] for g in got]), np.stack([g[1] for g in got])
    for name, a, b in (("cos", got_c, want_c), ("sin", got_s, want_s)):
        ulps = np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))
        same_sign = np.sign(a) == np.sign(b)
        ok = (ulps <= 1) & same_sign | (np.abs(a - b) <= np.spacing(np.float32(0)) )
        assert ok.all(), (name, np.argwhere(~ok)[:5], a[~ok][:5], b[~ok][:5])


# ------------------------------------------------------------------------------------------------ prefixes
class _Tok:
    """records the texts it encodes; one token per character"""
    def __init__(self, flat=True):
        self.seen = []
        if flat:
            self.encode_batch_flat = self._flat

    def encode_batch(self, texts):
        self.seen += texts
        return [np.arange(len(t), dtype=np.int32) for t in texts]

    def _flat(self, texts):
        toks = self.encode_batch(texts)
        offs = np.concatenate([[0], np.cumsum([len(t) for t in toks])]).astype(np.int32)
        return np.concatenate(toks), offs


class _Emb:
    def embed(self, toks):
        return np.zeros((len(toks), 4), np.float32)

    def embed_flat(self, flat, offs):
        return np.zeros((len(offs) - 1, 4), np.float32)


def _embedding(query, text, flat=True, max_batch_tokens=65536):
    import threading
    ge = object.__new__(E.GpuBertEmbedding)
    ge.tokenizer, ge._emb, ge._mu = _Tok(flat), _Emb(), threading.Lock()
    ge.query_instruction, ge.text_instruction, ge.max_batch_tokens, ge.dim = query, text, max_batch_tokens, 4
    return ge


@pytest.mark.parametrize("path", ["flat", "no flat encoder", "over the token budget", "single query"])
def test_queries_carry_only_the_query_prefix(path):
    ge = _embedding("search_query: ", "search_document: ", flat=path != "no flat encoder",
                    max_batch_tokens=4 if path == "over the token budget" else 65536)
    if path == "single query":
        ge.get_query_embedding("what is rope")
    else:
        ge.get_query_embedding_batch(["what is rope", "why gate"])
    assert ge.tokenizer.seen and all(t.startswith("search_query: ") and "search_document" not in t for t in ge.tokenizer.seen)


def test_documents_carry_only_the_document_prefix():
    ge = _embedding("search_query: ", "search_document: ")
    ge.get_text_embedding_batch(["rotary positions", "a gated ffn"])
    ge.get_text_embedding("one more")
    assert ge.tokenizer.seen == ["search_document: rotary positions", "search_document: a gated ffn", "search_document: one more"]


def test_models_without_a_document_prefix_embed_texts_as_they_are():
    ge = _embedding(None, None)
    ge.get_text_embedding_batch(["a b"])
    ge.get_query_embedding_batch(["c"])
    ge.get_query_embedding("d")
    assert ge.tokenizer.seen == ["a b", "c", "d"]
