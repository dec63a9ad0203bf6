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
    d, heads, inter = cfg.get("hidden_size"), cfg.get("num_attention_heads"), cfg.get("intermediate_size")
    if not all(isinstance(v, int) and v > 0 for v in (d, heads, inter)):
        raise ValueError(f"{cpath}: hidden_size, num_attention_heads and intermediate_size must be positive integers")
    if d % heads or d // heads not in (32, 64):
        raise ValueError(f"{cpath}: hidden_size {d} / num_attention_heads {heads}: K5 runs attention heads of 32 or 64 dims")
    if d % 128 or d > 1024:
        raise ValueError(f"{cpath}: hidden_size {d}: K5 runs multiples of 128 up to 1024")
    if inter % 128:
        raise ValueError(f"{cpath}: intermediate_size {inter}: K5 runs multiples of 128")
    return d


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
      cls_token, sep_token, unk_token   tokenizer_config.json's specials (default <s>, </s>, [UNK]), each in vocab.txt"""
    join = os.path.join
    cpath = join(model_dir, "config.json")
    try:
        peek = _json(cpath, required=False)
    except ValueError:
        peek = None
    mpnet = isinstance(peek, dict) and peek.get("model_type") == "mpnet"
    if mpnet:
        _check_mpnet_config(cpath, peek)
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

    cfg = _json(cpath)
    d = check_bert_config(cpath, cfg, "mpnet" if mpnet else "bert")
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
        raise ValueError(f"{where} {max_length!r}: must be an integer in [2, {bound}]")
    vpath = join(model_dir, "vocab.txt")
    if not os.path.isfile(vpath):
        raise ValueError(f"{vpath}: file missing (K5 takes WordPiece vocabularies)")
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
    LlamaIndex adds for BAAI/bge-* models [3P-unverified]."""

    def __init__(self, engine, tokenizer, config: dict, state_dict: dict, query_instruction: str | None = BGE_QUERY_INSTRUCTION,
                 max_batch_tokens: int = 65536, pooling: str = "cls", position_offset: int = 0):
        """position_offset: the position row of a sequence's first token (MPNet: 2)"""
        from . import _native
        if pooling not in ("cls", "mean"):
            raise ValueError(f"pooling {pooling!r}: expected 'cls' or 'mean'")
        self.tokenizer, self.query_instruction, self.max_batch_tokens = tokenizer, query_instruction, max_batch_tokens
        self.dim, self.pooling = config["hidden_size"], pooling
        self._emb = _native.Embedder(engine, config["num_hidden_layers"], config["hidden_size"], config["num_attention_heads"],
                                     config["intermediate_size"], config["vocab_size"], config.get("max_position_embeddings", 512),
                                     config.get("type_vocab_size", 2), config.get("layer_norm_eps", 1e-12))
        if pooling == "mean":
            self._emb.set_pooling(_native.POOL_MEAN)
        if position_offset:
            self._emb.set_position_offset(position_offset)
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
        return self._embed_tokens(self.tokenizer.encode_batch(list(texts)))

    def get_text_embedding(self, text: str):
        return self.get_text_embedding_batch([text])[0]

    def get_query_embedding(self, query: str):
        return self.get_text_embedding((self.query_instruction or "") + query)

    def get_query_embedding_batch(self, queries):
        """one K5 forward for a coalesced batch of queries (kaito_b200.batcher); the token ids stay packed numpy arrays from
        the native tokeniser to the embedder's C entry point"""
        texts = [(self.query_instruction or "") + q for q in queries]
        if hasattr(self.tokenizer, "encode_batch_flat"):
            flat, offs = self.tokenizer.encode_batch_flat(texts)
            if len(flat) <= self.max_batch_tokens:
                with self._mu:
                    return self._emb.embed_flat(flat, offs)
        return self.get_text_embedding_batch(texts)


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
