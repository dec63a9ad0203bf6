"""Embedding-model interface of the host (mirrors embedding/base.py:21-31 BaseEmbeddingModel).
`GpuBertEmbedding` is the production embedder for the CRD's `embedding.local.modelID` (K5, the BERT forward in
libkaito_rag; SURVEY.md section 8 a5); `HashingEmbedding` is a deterministic stand-in without weights for the host-logic
tests (no checkpoints are available offline) and never the default of the service."""
from __future__ import annotations

import hashlib
import json
import os
import re

import numpy as np


class BaseEmbeddingModel:
    def get_text_embedding(self, text: str) -> list[float]:
        raise NotImplementedError

    def get_text_embedding_batch(self, texts: list[str]) -> np.ndarray:
        return np.asarray([self.get_text_embedding(t) for t in texts], np.float32)

    def get_query_embedding(self, query: str) -> list[float]:
        return self.get_text_embedding(query)

    def get_embedding_dimension(self) -> int:
        """reference probes by embedding a dummy sentence (huggingface_local_embedding.py:55-61)"""
        return len(self.get_text_embedding("dimension probe"))


class HashingEmbedding(BaseEmbeddingModel):
    """Unit-norm sum of per-word pseudo-random Gaussian vectors (seeded by sha256 of the word):
    deterministic, no weights, texts sharing words are close.  NOT a language model."""

    def __init__(self, dim: int = 384):
        self.dim = dim
        self._cache: dict[str, np.ndarray] = {}

    def _word(self, w: str) -> np.ndarray:
        v = self._cache.get(w)
        if v is None:
            seed = int.from_bytes(hashlib.sha256(w.encode()).digest()[:8], "little")
            v = np.random.default_rng(seed).standard_normal(self.dim).astype(np.float32)
            self._cache[w] = v
        return v

    def get_text_embedding(self, text: str):
        words = re.findall(r"\w+", text.lower()) or [""]
        v = np.sum([self._word(w) for w in words], axis=0)
        n = float(np.linalg.norm(v))
        return (v / n if n > 0 else v).astype(np.float32)

    def get_embedding_dimension(self) -> int:
        return self.dim


BGE_QUERY_INSTRUCTION = "Represent this question for searching relevant passages: "

_ST_MODULE = "sentence_transformers.models."
_POOLING_FLAGS = ("pooling_mode_cls_token", "pooling_mode_mean_tokens", "pooling_mode_max_tokens",
                  "pooling_mode_mean_sqrt_len_tokens", "pooling_mode_weightedmean_tokens", "pooling_mode_lasttoken")


def _json(path: str, required: bool = True):
    if not os.path.isfile(path):
        if required:
            raise ValueError(f"{path}: file missing")
        return None
    try:
        with open(path, encoding="utf-8") as f:
            return json.load(f)
    except (OSError, ValueError) as e:
        raise ValueError(f"{path}: unreadable ({e})") from None


def check_bert_config(cpath: str, cfg: dict, model_type: str = "bert") -> int:
    """the encoder shapes K5 runs (config.json at cpath, parsed as cfg, of a `model_type` encoder: "bert" or "mpnet");
    returns hidden_size or raises a ValueError naming the file and field (shared by the embedder and cross-encoder snapshot
    readers)"""
    for field, want, default in (("model_type", model_type, None), ("position_embedding_type", "absolute", "absolute"),
                                 ("hidden_act", "gelu", "gelu"), ("is_decoder", False, False)):
        if cfg.get(field, default) != want:
            raise ValueError(f"{cpath}: {field} {cfg.get(field, default)!r}: K5 runs {field} {want!r} only")
    return _check_shapes(cpath, cfg)


def _check_shapes(cpath: str, cfg: dict, names=("hidden_size", "num_attention_heads", "intermediate_size")) -> int:
    """K5's shape rules on a config with BERT field names; `names` are the fields the file states them under"""
    d, heads, inter = cfg.get("hidden_size"), cfg.get("num_attention_heads"), cfg.get("intermediate_size")
    if not all(isinstance(v, int) and v > 0 for v in (d, heads, inter)):
        raise ValueError(f"{cpath}: {', '.join(names[:2])} and {names[2]} must be positive integers")
    d_name, h_name, i_name = names
    if d % heads or d // heads not in (32, 64):
        raise ValueError(f"{cpath}: {d_name} {d} / {h_name} {heads}: K5 runs attention heads of 32 or 64 dims")
    if d % 128 or d > 1024:
        raise ValueError(f"{cpath}: {d_name} {d}: K5 runs multiples of 128 up to 1024")
    if inter % 128:
        raise ValueError(f"{cpath}: {i_name} {inter}: K5 runs multiples of 128")
    return d


# nomic-embed-text v1 / v1.5 (model_type "nomic_bert"): a post-LN BERT with rotary positions, a SwiGLU FFN and no Linear
# biases.  Its config.json comes in two forms: the hub's custom-code names (n_embd, ...) [3P-unverified: no snapshot can be
# downloaded here] and transformers' NomicBertConfig names (hidden_size, ..., rope_parameters).
NOMIC_QUERY_PREFIX = "search_query: "          # the model card's task prefixes [3P-unverified whether LlamaIndex adds them]
NOMIC_DOCUMENT_PREFIX = "search_document: "
# hub field -> K5's BERT field
_NOMIC_HUB_SHAPES = (("n_layer", "num_hidden_layers"), ("n_embd", "hidden_size"), ("n_head", "num_attention_heads"),
                     ("n_inner", "intermediate_size"), ("n_positions", "max_position_embeddings"), ("vocab_size", "vocab_size"))
# hub flags whose absence means what K5 runs
_NOMIC_HUB_FLAGS = (("rotary_emb_interleaved", False), ("rotary_scaling_factor", None), ("prenorm", False),
                    ("use_rms_norm", False), ("causal", False))


def _nomic_config(cpath: str, cfg: dict) -> dict:
    """a nomic_bert config.json in either form as K5's BERT-named config plus "rotary_base", or a ValueError naming the file
    and field.  K5 runs rotary fraction 1.0, not interleaved, without scaling, a SwiGLU FFN, no biases, post-LN LayerNorm,
    bidirectional attention."""
    def need(field, ok, what):
        if field not in cfg:
            raise ValueError(f"{cpath}: {field} missing: a nomic_bert config must state it ({what})")
        if not ok(cfg[field]):
            raise ValueError(f"{cpath}: {field} {cfg[field]!r}: K5 runs {what} only")
        return cfg[field]

    num = lambda v: isinstance(v, (int, float)) and not isinstance(v, bool)   # noqa: E731
    if "n_embd" in cfg:                          # the hub's custom-code config
        out = {k5: cfg.get(hub) for hub, k5 in _NOMIC_HUB_SHAPES}
        for hub, k5 in _NOMIC_HUB_SHAPES:
            need(hub, lambda v: isinstance(v, int) and not isinstance(v, bool) and v > 0, "a positive integer")
        need("rotary_emb_fraction", lambda v: num(v) and v == 1.0, "rotary_emb_fraction 1.0 (every head dim rotated)")
        base = need("rotary_emb_base", lambda v: num(v) and v > 0, "a positive rotary_emb_base")
        for field, want in _NOMIC_HUB_FLAGS:
            if cfg.get(field, want) != want:
                why = " (dynamic NTK scaling makes an embedding depend on the batch's padded length)" \
                    if field == "rotary_scaling_factor" else ""
                raise ValueError(f"{cpath}: {field} {cfg[field]!r}: K5 runs {field} {want!r} only{why}")
        need("activation_function", lambda v: v == "swiglu", "activation_function 'swiglu'")
        for field in ("qkv_proj_bias", "mlp_fc1_bias", "mlp_fc2_bias"):
            need(field, lambda v: v is False, f"{field} false (no Linear biases)")
        eps = need("layer_norm_epsilon", lambda v: num(v) and v > 0, "a positive layer_norm_epsilon")
        names = ("n_embd", "n_head", "n_inner")
    else:                                        # transformers' NomicBertConfig
        out = {k: cfg.get(k) for k in ("num_hidden_layers", "hidden_size", "num_attention_heads", "intermediate_size",
                                       "max_position_embeddings", "vocab_size")}
        for k in out:
            need(k, lambda v: isinstance(v, int) and not isinstance(v, bool) and v > 0, "a positive integer")
        need("hidden_act", lambda v: v == "silu", "hidden_act 'silu' (the gated FFN)")
        rp = need("rope_parameters", lambda v: isinstance(v, dict), "rope_parameters {'rope_type': 'default', 'rope_theta': ...}")
        if rp.get("rope_type", "default") != "default":
            raise ValueError(f"{cpath}: rope_parameters.rope_type {rp['rope_type']!r}: K5 runs 'default' RoPE only (dynamic "
                             "NTK scaling makes an embedding depend on the batch's padded length)")
        base = rp.get("rope_theta")
        if not (num(base) and base > 0):
            raise ValueError(f"{cpath}: rope_parameters.rope_theta {base!r}: K5 runs a positive rotary base only")
        hd = cfg.get("head_dim")
        if hd is not None and hd * out["num_attention_heads"] != out["hidden_size"]:
            raise ValueError(f"{cpath}: head_dim {hd!r}: K5 runs head_dim = hidden_size / num_attention_heads only")
        if cfg.get("is_decoder", False):
            raise ValueError(f"{cpath}: is_decoder {cfg['is_decoder']!r}: K5 runs bidirectional encoders only")
        eps = cfg.get("layer_norm_eps", 1e-12)
        names = ("hidden_size", "num_attention_heads", "intermediate_size")
    _check_shapes(cpath, out, names)
    tv = cfg.get("type_vocab_size", 2)
    if not (isinstance(tv, int) and tv >= 1):
        raise ValueError(f"{cpath}: type_vocab_size {tv!r}: must be a positive integer")
    return dict(out, type_vocab_size=tv, layer_norm_eps=float(eps), rotary_base=float(base))


# nomic tensor names (hub checkpoint and transformers' NomicBertModel) -> the BertModel names K5 loads; the gate projection
# (fc12 / gate_proj) becomes intermediate.gate, the up projection (fc11 / up_proj) intermediate.dense
_NOMIC_NAMES = ((r"^emb_ln\.", "embeddings.LayerNorm."), (r"^(?:encoder\.layers|layers)\.(\d+)\.", r"encoder.layer.\1."),
                (r"\.(?:attn\.out_proj|self_attn\.o_proj)\.", ".attention.output.dense."),
                (r"\.self_attn\.q_proj\.", ".attention.self.query."), (r"\.self_attn\.k_proj\.", ".attention.self.key."),
                (r"\.self_attn\.v_proj\.", ".attention.self.value."),
                (r"\.mlp\.(?:fc11|up_proj)\.", ".intermediate.dense."), (r"\.mlp\.(?:fc12|gate_proj)\.", ".intermediate.gate."),
                (r"\.mlp\.(?:fc2|down_proj)\.", ".output.dense."),
                (r"\.(?:norm1|post_attention_layernorm)\.", ".attention.output.LayerNorm."),
                (r"\.(?:norm2|post_mlp_layernorm)\.", ".output.LayerNorm."))
_NOMIC_WQKV = re.compile(r"^(encoder\.layer\.\d+)\.attn\.Wqkv\.(weight|bias)$")


def nomic_state(state: dict, cfg: dict) -> dict:
    """a nomic checkpoint's tensors (either name set, without a model prefix) under K5's names: Wqkv [3 hidden, hidden]
    split into Q, K, V rows (transformers' Chunk(dim=0)); zero biases for every Linear (nomic has none: adding +0.0 changes
    no bit) and a zero token-type row when the checkpoint has no table; rotary inv_freq buffers dropped.  cfg: _nomic_config's"""
    out = {}
    for k, v in state.items():
        if k.endswith("inv_freq"):
            continue
        for a, b in _NOMIC_NAMES:
            k = re.sub(a, b, k)
        m = _NOMIC_WQKV.match(k)
        if m:
            for part, nm in zip(np.split(np.asarray(v), 3, axis=0), ("query", "key", "value")):
                out[f"{m.group(1)}.attention.self.{nm}.{m.group(2)}"] = part
            continue
        out[k] = v
    d, inter = cfg["hidden_size"], cfg["intermediate_size"]
    for l in range(cfg["num_hidden_layers"]):
        p = f"encoder.layer.{l}."
        for nm, n in (("attention.self.query", d), ("attention.self.key", d), ("attention.self.value", d),
                      ("attention.output.dense", d), ("intermediate.dense", inter), ("intermediate.gate", inter), ("output.dense", d)):
            out.setdefault(p + nm + ".bias", np.zeros(n, np.float32))
    if "embeddings.token_type_embeddings.weight" not in out:
        out["embeddings.token_type_embeddings.weight"] = np.zeros((1, d), np.float32)
    return out


# transformers MPNetModel names -> the BertModel names K5 loads (encoder.relative_attention_bias.weight keeps its name)
_MPNET_NAMES = ((".attention.attn.q.", ".attention.self.query."), (".attention.attn.k.", ".attention.self.key."),
                (".attention.attn.v.", ".attention.self.value."), (".attention.attn.o.", ".attention.output.dense."),
                (".attention.LayerNorm.", ".attention.output.LayerNorm."))
MPNET_REL_BIAS = "encoder.relative_attention_bias.weight"
MPNET_BUCKETS = 32            # transformers' MPNetEncoder computes 32 relative-position buckets whatever the config says
MPNET_POSITION_OFFSET = 2     # MPNet numbers positions from padding_idx + 1, padding_idx = 1


def _k5_name(k: str) -> str:
    """a checkpoint tensor name without its "bert." / "mpnet." prefix, MPNet names mapped onto BERT's"""
    for prefix in ("bert.", "mpnet."):
        if k.startswith(prefix):
            k = k[len(prefix):]
            break
    for a, b in _MPNET_NAMES:
        k = k.replace(a, b)
    return k


def load_state(model_dir: str) -> dict:
    """model.safetensors or pytorch_model.bin of a snapshot as numpy fp32 arrays, names without the "bert." / "mpnet."
    prefix; MPNet's attention names are mapped onto BERT's (attention.attn.q -> attention.self.query, ...)"""
    st_path, bin_path = os.path.join(model_dir, "model.safetensors"), os.path.join(model_dir, "pytorch_model.bin")
    if os.path.exists(st_path):
        from safetensors.numpy import load_file
        state = load_file(st_path)
    elif os.path.exists(bin_path):
        import torch
        state = {k: v.float().numpy() for k, v in torch.load(bin_path, map_location="cpu").items()}
    else:
        raise ValueError(f"{model_dir}: neither model.safetensors nor pytorch_model.bin")
    return {_k5_name(k): v for k, v in state.items()}


def _check_mpnet_config(cpath: str, cfg: dict):
    """what an MPNet config.json must state before anything else of the snapshot is read"""
    nb = cfg.get("relative_attention_num_buckets")
    if nb != MPNET_BUCKETS:
        raise ValueError(f"{cpath}: model_type 'mpnet' with relative_attention_num_buckets {nb!r}: K5 runs MPNet encoders that "
                         f"state {MPNET_BUCKETS} buckets (transformers always computes {MPNET_BUCKETS})")


def _special(tc: dict, field: str, default: str) -> str:
    """a special token of tokenizer_config.json: a string or an AddedToken dict {"content": ...}"""
    v = tc.get(field, default)
    return v.get("content", default) if isinstance(v, dict) else v


def read_snapshot_spec(model_dir: str) -> dict:
    """What sentence-transformers would compute from a model snapshot, or a ValueError naming the file and field that asks for
    something K5 does not compute.  Reads JSON only (no weights, no GPU).  Returns
      pooling            "cls" | "mean"   (modules.json + <Pooling path>/config.json; no modules.json: "cls")
      max_length         tokens per sequence incl. [CLS] / [SEP] (sentence_bert_config.json max_seq_length, else
                         min(tokenizer_config.json model_max_length, config.json max_position_embeddings), else 512)
      do_lower_case      tokenizer_config.json do_lower_case (default true)
      query_instruction  the bge prefix for CLS-pooled BERT snapshots, None for mean-pooled and MPNet ones [3P-unverified]
    and for config.json model_type "mpnet" (all-mpnet-base-v2, multi-qa-mpnet-*) also
      model_type         "mpnet"
      position_offset    2 (MPNet's first position row)
      cls_token, sep_token, unk_token   tokenizer_config.json's specials (default <s>, </s>, [UNK]), each in vocab.txt
    and for config.json model_type "nomic_bert" (nomic-embed-text-v1 / -v1.5; either config form, see _nomic_config)
      model_type         "nomic_bert"
      query_instruction  "search_query: ", text_instruction "search_document: " (the model card's task prefixes)
      config             the config under BERT names, max_position_embeddings = n_positions, plus rotary_base"""
    join = os.path.join
    cpath = join(model_dir, "config.json")
    try:
        peek = _json(cpath, required=False)
    except ValueError:
        peek = None
    mpnet = isinstance(peek, dict) and peek.get("model_type") == "mpnet"
    nomic = isinstance(peek, dict) and peek.get("model_type") == "nomic_bert"
    if mpnet:
        _check_mpnet_config(cpath, peek)
    if nomic:
        ncfg = _nomic_config(cpath, peek)
    pooling = "cls"
    mpath = join(model_dir, "modules.json")
    modules = _json(mpath, required=False)
    if modules is not None:
        types = [m.get("type", "") if isinstance(m, dict) else "" for m in modules] if isinstance(modules, list) else []
        names = [t[len(_ST_MODULE):] if t.startswith(_ST_MODULE) else t for t in types]
        if names[:2] != ["Transformer", "Pooling"] or names[2:] not in ([], ["Normalize"]):
            raise ValueError(f"{mpath}: modules {types}: supported are a Transformer, then a Pooling, then an optional "
                             "Normalize (a Dense head or any other module is not)")
        if modules[0].get("path", "") != "":
            raise ValueError(f"{mpath}: the Transformer's path is {modules[0]['path']!r}: the model must be at the snapshot root")
        ppath = join(model_dir, modules[1].get("path", ""), "config.json")
        pc = _json(ppath)
        on = [k for k in _POOLING_FLAGS if pc.get(k)]
        if on not in (["pooling_mode_cls_token"], ["pooling_mode_mean_tokens"]):
            raise ValueError(f"{ppath}: pooling modes {on}: exactly one of pooling_mode_cls_token or pooling_mode_mean_tokens "
                             "must be true (max, mean_sqrt_len, weightedmean, lasttoken and combinations are not supported)")
        if pc.get("include_prompt", True) is not True:
            raise ValueError(f"{ppath}: include_prompt {pc['include_prompt']!r}: only true (pool over every token) is supported")
        pooling = "cls" if on[0] == "pooling_mode_cls_token" else "mean"

    cfg = ncfg if nomic else _json(cpath)
    d = cfg["hidden_size"] if nomic else check_bert_config(cpath, cfg, "mpnet" if mpnet else "bert")
    if modules is not None and pc.get("word_embedding_dimension", d) != d:
        raise ValueError(f"{ppath}: word_embedding_dimension {pc['word_embedding_dimension']} differs from config.json "
                         f"hidden_size {d}")
    max_pos = cfg.get("max_position_embeddings", 512)
    off = MPNET_POSITION_OFFSET if mpnet else 0
    max_tok = max_pos - off                  # positions off .. max_pos - 1

    tpath = join(model_dir, "tokenizer_config.json")
    tc = _json(tpath, required=False) or {}
    do_lower_case = tc.get("do_lower_case", True)
    spath = join(model_dir, "sentence_bert_config.json")
    sbc = _json(spath, required=False) or {}
    if sbc.get("do_lower_case") and not do_lower_case:
        raise ValueError(f"{spath}: do_lower_case true with a cased tokenizer ({tpath} do_lower_case false) is not supported")
    if sbc.get("max_seq_length") is not None:
        max_length, where = sbc["max_seq_length"], f"{spath}: max_seq_length"
    else:
        max_length, where = min(tc.get("model_max_length", max_tok), max_tok), f"{tpath}: model_max_length"
    if not isinstance(max_length, int) or not 2 <= max_length <= max_tok:
        bound = f"config.json max_position_embeddings {max_pos} - {off}" if off else f"config.json max_position_embeddings {max_pos}"
        if nomic and "n_positions" in peek:
            bound = f"config.json n_positions {max_pos}"
        raise ValueError(f"{where} {max_length!r}: must be an integer in [2, {bound}]")
    vpath = join(model_dir, "vocab.txt")
    if not os.path.isfile(vpath):
        raise ValueError(f"{vpath}: file missing (K5 takes WordPiece vocabularies)")
    if nomic:
        return {"pooling": pooling, "max_length": max_length, "do_lower_case": bool(do_lower_case),
                "query_instruction": NOMIC_QUERY_PREFIX, "text_instruction": NOMIC_DOCUMENT_PREFIX, "model_type": "nomic_bert",
                "config": ncfg}
    if not mpnet:
        return {"pooling": pooling, "max_length": max_length, "do_lower_case": bool(do_lower_case),
                "query_instruction": BGE_QUERY_INSTRUCTION if pooling == "cls" else None}
    specials = {f: _special(tc, f, dv) for f, dv in (("cls_token", "<s>"), ("sep_token", "</s>"), ("unk_token", "[UNK]"))}
    with open(vpath, encoding="utf-8") as f:
        vocab = {line.rstrip("\n") for line in f}
    for field, tok in specials.items():
        if not isinstance(tok, str) or tok not in vocab:
            raise ValueError(f"{vpath}: {tpath} {field} {tok!r} is not a token of the vocabulary")
    return dict({"pooling": pooling, "max_length": max_length, "do_lower_case": bool(do_lower_case), "query_instruction": None,
                 "model_type": "mpnet", "position_offset": MPNET_POSITION_OFFSET}, **specials)


class GpuBertEmbedding(BaseEmbeddingModel):
    """BERT and MPNet sentence embedders (bge, all-MiniLM, e5, gte, all-mpnet, ...) on the GPU (K5, kaito_b200/csrc/embed.cu): WordPiece on the
    host, BERT encoder forward + CLS or mean pooling + L2 normalisation in libkaito_rag.  Mirrors
    LocalHuggingFaceEmbedding (embedding/huggingface_local_embedding.py:31-61); from_pretrained reads the pooling, casing
    and length from the snapshot (read_snapshot_spec).  CLS-pooled snapshots' queries get the bge instruction prefix
    LlamaIndex adds for BAAI/bge-* models [3P-unverified].  nomic-embed-text (nomic_bert) snapshots run rotary positions and
    the gated FFN, and their queries / documents get the model card's "search_query: " / "search_document: " prefixes."""

    def __init__(self, engine, tokenizer, config: dict, state_dict: dict, query_instruction: str | None = BGE_QUERY_INSTRUCTION,
                 max_batch_tokens: int = 65536, pooling: str = "cls", position_offset: int = 0, text_instruction: str | None = None,
                 rotary_base: float = 0.0):
        """position_offset: the position row of a sequence's first token (MPNet: 2); text_instruction: the prefix of every
        document text (nomic: "search_document: "; queries take query_instruction alone); rotary_base > 0: rotary positions
        instead of a position table (nomic)"""
        from . import _native
        if pooling not in ("cls", "mean"):
            raise ValueError(f"pooling {pooling!r}: expected 'cls' or 'mean'")
        self.tokenizer, self.query_instruction, self.max_batch_tokens = tokenizer, query_instruction, max_batch_tokens
        self.text_instruction = text_instruction
        self.dim, self.pooling = config["hidden_size"], pooling
        self._emb = _native.Embedder(engine, config["num_hidden_layers"], config["hidden_size"], config["num_attention_heads"],
                                     config["intermediate_size"], config["vocab_size"], config.get("max_position_embeddings", 512),
                                     config.get("type_vocab_size", 2), config.get("layer_norm_eps", 1e-12))
        if pooling == "mean":
            self._emb.set_pooling(_native.POOL_MEAN)
        if position_offset:
            self._emb.set_position_offset(position_offset)
        if rotary_base:
            self._emb.set_rotary(rotary_base)
        self._emb.load_state_dict(state_dict)
        import threading
        self._mu = threading.Lock()          # one forward at a time: the embedder owns one set of activation buffers

    @classmethod
    def from_pretrained(cls, engine, model_dir: str, **kw):
        """model_dir: a Hugging Face / sentence-transformers snapshot (config.json, vocab.txt, model.safetensors or
        pytorch_model.bin; modules.json, the Pooling config, sentence_bert_config.json and tokenizer_config.json when
        present).  Raises ValueError before any weight is read when the snapshot asks for what K5 does not compute.
        MPNet snapshots: the weights are loaded under K5's BERT names with a zero token-type row (adding +0.0 changes no
        bit), positions start at row 2 and the tokenizer takes the snapshot's <s> / </s> / [UNK]."""
        from .text import WordPieceTokenizer
        spec = read_snapshot_spec(model_dir)
        cfg = _json(os.path.join(model_dir, "config.json"))
        state = load_state(model_dir)
        kw.setdefault("query_instruction", spec["query_instruction"])
        kw.setdefault("pooling", spec["pooling"])
        specials = {}
        if spec.get("model_type") == "nomic_bert":
            cfg = spec["config"]
            state = nomic_state(state, cfg)
            cfg = dict(cfg, type_vocab_size=state["embeddings.token_type_embeddings.weight"].shape[0])
            kw.setdefault("text_instruction", spec["text_instruction"])
            kw.setdefault("rotary_base", cfg["rotary_base"])
        if spec.get("model_type") == "mpnet":
            if MPNET_REL_BIAS not in state:
                raise ValueError(f"{model_dir}: model_type 'mpnet' without the tensor {MPNET_REL_BIAS}")
            cfg = dict(cfg, type_vocab_size=1)
            state = dict(state, **{"embeddings.token_type_embeddings.weight": np.zeros((1, cfg["hidden_size"]), np.float32)})
            kw.setdefault("position_offset", spec["position_offset"])
            specials = {k: spec[k] for k in ("cls_token", "sep_token", "unk_token")}
        tok = WordPieceTokenizer.from_file(os.path.join(model_dir, "vocab.txt"), do_lower_case=spec["do_lower_case"],
                                           max_length=spec["max_length"], **specials)
        return cls(engine, tok, cfg, state, **kw)

    def get_embedding_dimension(self) -> int:
        return self.dim

    def _embed_tokens(self, token_lists):
        import numpy as np
        out, batch, ntok = [], [], 0
        for t in token_lists:
            if batch and ntok + len(t) > self.max_batch_tokens:
                with self._mu:
                    out.append(self._emb.embed(batch))
                batch, ntok = [], 0
            batch.append(t); ntok += len(t)
        if batch:
            with self._mu:
                out.append(self._emb.embed(batch))
        return np.concatenate(out)

    def get_text_embedding_batch(self, texts):
        """documents: each text behind text_instruction (None: as it is)"""
        texts = [self.text_instruction + t for t in texts] if self.text_instruction else list(texts)
        return self._embed_tokens(self.tokenizer.encode_batch(texts))

    def get_text_embedding(self, text: str):
        return self.get_text_embedding_batch([text])[0]

    def get_query_embedding(self, query: str):
        return self._embed_tokens(self.tokenizer.encode_batch([(self.query_instruction or "") + query]))[0]

    def get_query_embedding_batch(self, queries):
        """one K5 forward for a coalesced batch of queries (kaito_b200.batcher); the token ids stay packed numpy arrays from
        the native tokeniser to the embedder's C entry point.  Queries take query_instruction only, never text_instruction."""
        texts = [(self.query_instruction or "") + q for q in queries]
        if hasattr(self.tokenizer, "encode_batch_flat"):
            flat, offs = self.tokenizer.encode_batch_flat(texts)
            if len(flat) <= self.max_batch_tokens:
                with self._mu:
                    return self._emb.embed_flat(flat, offs)
        return self._embed_tokens(self.tokenizer.encode_batch(texts))


class RemoteEmbeddingModel(BaseEmbeddingModel):
    """`embedding.remote` of the CRD (embedding/remote_embedding.py:24-76): POST {"inputs": text} with a bearer token to
    REMOTE_EMBEDDING_URL, the reply is the embedding as a JSON list.  Host-side HTTP only -- the retrieval kernels take the
    vectors exactly as with the local model."""

    def __init__(self, model_url: str, api_key: str, transport=None):
        self.model_url, self.api_key, self._transport = model_url, api_key, transport
        self._client = None

    def _http(self):
        if self._client is None:
            import httpx
            kw = {"transport": self._transport} if self._transport is not None else {}
            self._client = httpx.Client(timeout=300.0, **kw)
        return self._client

    def get_text_embedding(self, text: str):
        import httpx
        headers = {"Authorization": f"Bearer {self.api_key}", "Content-Type": "application/json"}
        try:
            r = self._http().post(self.model_url, headers=headers, json={"inputs": text})
            r.raise_for_status()
            emb = r.json()
        except httpx.HTTPError as e:
            raise RuntimeError(f"Failed to get embedding from remote model: {e}")
        if not isinstance(emb, list):
            raise ValueError("Unexpected response format. Expected a list.")
        return np.asarray(emb, np.float32)

    def get_embedding_dimension(self) -> int:
        return len(self.get_text_embedding("This is a dummy sentence."))
