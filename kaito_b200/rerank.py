"""Cross-encoder reranking of /retrieve candidates: a BERT cross-encoder (BertForSequenceClassification with one label, e.g.
cross-encoder/ms-marco-MiniLM-L-6-v2) scores each (query, passage) pair on the GPU -- the K5 encoder with token types for the
second segment, the pooler and classifier head, and a per-query top-k selection, all in libkaito_rag (kaito_b200/csrc/embed.cu).
The hybrid stage hands over N = min(max(top_k, KRAG_RERANK_CANDIDATES), RAG_MAX_TOP_K) fused candidates per query and the
reranker keeps the top_k best (LlamaIndex's retriever similarity_top_k, then the postprocessor's top_n)."""
from __future__ import annotations

import os
import threading

import numpy as np

from .embedding import _json, check_bert_config, load_state

RERANK_CANDIDATES = 30           # KRAG_RERANK_CANDIDATES default
_ACTIVATIONS = {"Sigmoid": "sigmoid", "Identity": "identity"}
PRECISIONS = ("fp32", "fp16")    # KRAG_RERANK_PRECISION; the default is the fp32-accurate forward


def precision_from_env() -> str:
    """KRAG_RERANK_PRECISION: "fp32" (default) or "fp16"; a ValueError for anything else"""
    p = os.getenv("KRAG_RERANK_PRECISION") or "fp32"
    if p not in PRECISIONS:
        raise ValueError(f"KRAG_RERANK_PRECISION {p!r}: expected 'fp32' or 'fp16'")
    return p


def read_cross_encoder_spec(model_dir: str) -> dict:
    """What sentence-transformers' CrossEncoder computes from a snapshot, or a ValueError naming the file and field that asks
    for something K5 does not compute.  Reads JSON only (no weights, no GPU).  Returns
      max_length     tokens per pair incl. [CLS] / [SEP] / [SEP]: tokenizer_config.json model_max_length, else
                     config.json max_position_embeddings (default 512); a limit beyond the position table is refused
      do_lower_case  tokenizer_config.json do_lower_case (default true)
      activation     "sigmoid" | "identity": config.json sentence_transformers.activation_fn or the legacy
                     sbert_ce_default_activation_function; Sigmoid when neither is given (the default for one label)
                     [3P-unverified]"""
    join = os.path.join
    cpath = join(model_dir, "config.json")
    cfg = _json(cpath)
    check_bert_config(cpath, cfg)
    archs = cfg.get("architectures") or []
    if "BertForSequenceClassification" not in archs:
        raise ValueError(f"{cpath}: architectures {archs!r}: a cross-encoder is a BertForSequenceClassification")
    labels = len(cfg["id2label"]) if isinstance(cfg.get("id2label"), dict) else cfg.get("num_labels", 2)
    if labels != 1:
        raise ValueError(f"{cpath}: {labels} labels (num_labels / id2label): K5 reranks with one relevance logit only")
    if not isinstance(cfg.get("type_vocab_size", 2), int) or cfg.get("type_vocab_size", 2) < 2:
        raise ValueError(f"{cpath}: type_vocab_size {cfg.get('type_vocab_size')!r}: sentence pairs need token type 1")
    st = cfg.get("sentence_transformers") if isinstance(cfg.get("sentence_transformers"), dict) else {}
    fn = st.get("activation_fn") or cfg.get("sbert_ce_default_activation_function") or "torch.nn.modules.activation.Sigmoid"
    act = _ACTIVATIONS.get(str(fn).rsplit(".", 1)[-1]) if isinstance(fn, str) and fn.startswith("torch.nn.") else None
    if act is None:
        raise ValueError(f"{cpath}: activation function {fn!r}: K5 applies torch.nn Sigmoid or Identity only")
    max_pos = cfg.get("max_position_embeddings", 512)
    tpath = join(model_dir, "tokenizer_config.json")
    tc = _json(tpath, required=False) or {}
    mml = tc.get("model_max_length")
    if isinstance(mml, (int, float)) and not isinstance(mml, bool) and mml >= 1e12:
        mml = None                           # transformers' "no limit" sentinel (int(1e30))
    max_length = max_pos if mml is None else mml
    if not isinstance(max_length, int) or not 4 <= max_length <= max_pos:
        raise ValueError(f"{tpath}: model_max_length {max_length!r}: must be an integer in [4, config.json "
                         f"max_position_embeddings {max_pos}]")
    if not os.path.isfile(join(model_dir, "vocab.txt")):
        raise ValueError(f"{join(model_dir, 'vocab.txt')}: file missing (K5 takes WordPiece vocabularies)")
    return {"max_length": max_length, "do_lower_case": bool(tc.get("do_lower_case", True)), "activation": act}


def check_head_tensors(where: str, state: dict, hidden: int):
    """the classifier head a one-label BertForSequenceClassification carries (names without "bert."), or a ValueError
    naming the file and tensor"""
    for name, shape in (("pooler.dense.weight", (hidden, hidden)), ("pooler.dense.bias", (hidden,)),
                        ("classifier.weight", (1, hidden)), ("classifier.bias", (1,))):
        if name not in state:
            raise ValueError(f"{where}: tensor {name} missing (a cross-encoder carries the pooler and a one-label classifier)")
        if tuple(np.shape(state[name])) != shape:
            raise ValueError(f"{where}: tensor {name} has shape {tuple(np.shape(state[name]))}, expected {shape}")


def pair_lengths(n_q: int, n_d: int, max_length: int) -> tuple[int, int]:
    """tokens kept of each half of [CLS] q [SEP] d [SEP] under truncation="longest_first" to max_length: the rule of the
    Rust tokenizers' pair truncation (the shorter half stays whole when it fits in half the budget, else the budget is
    halved; on equal lengths the first half gets the smaller share) [3P-unverified]"""
    budget = max_length - 3
    if n_q + n_d <= budget:
        return n_q, n_d
    n1, n2, swap = n_q, n_d, n_q > n_d
    if swap:
        n1, n2 = n2, n1
    n2 = n1 if n1 > budget else max(n1, budget - n1)
    if n1 + n2 > budget:
        n1 = budget // 2
        n2 = n1 + budget % 2
    if swap:
        n1, n2 = n2, n1
    return min(n_q, n1), min(n_d, n2)


def build_pairs(cls_id: int, sep_id: int, queries: list[tuple[np.ndarray, int]], passages: list[list[tuple[np.ndarray, int]]],
                max_length: int):
    """packed pairs for krag_rerank: queries[i] = (ids, full length), passages[i] = that query's candidates as (ids cut at
    max_length - 3, full length).  Returns (flat int32 ids, token offsets [n_pairs + 1], seg_b [n_pairs], pair offsets
    [n_queries + 1])"""
    parts, lens, seg = [], [], []
    poff = np.zeros(len(queries) + 1, np.int32)
    head, mid = np.asarray([cls_id], np.int32), np.asarray([sep_id], np.int32)
    for i, ((q, nq), cands) in enumerate(zip(queries, passages)):
        for d, nd in cands:
            a, b = pair_lengths(nq, nd, max_length)
            parts += [head, q[:a], mid, d[:b], mid]
            lens.append(a + b + 3)
            seg.append(a + 2)
        poff[i + 1] = poff[i] + len(cands)
    toff = np.zeros(len(lens) + 1, np.int32)
    np.cumsum(lens, out=toff[1:])
    flat = np.concatenate(parts).astype(np.int32) if parts else np.zeros(0, np.int32)
    return flat, toff, np.asarray(seg, np.int32), poff


class GpuCrossEncoder:
    """A BERT cross-encoder on the GPU (krag_rerank).  rerank(queries, candidate ordinals per query, top_k, passages) scores
    every (query, passage) pair and returns the positions and scores of each query's top_k; `passages(ordinals, encode)` is the
    store's per-ordinal token cache (_IndexState.pair_passages), filled through `encode_passages` on a miss."""

    def __init__(self, engine, tokenizer, config: dict, state_dict: dict, max_length: int = 512, activation: str = "sigmoid",
                 precision: str = "fp32"):
        from . import _native
        if activation not in ("sigmoid", "identity"):
            raise ValueError(f"activation {activation!r}: expected 'sigmoid' or 'identity'")
        if precision not in PRECISIONS:
            raise ValueError(f"precision {precision!r}: expected 'fp32' or 'fp16'")
        self.tokenizer, self.max_length, self.activation, self.precision = tokenizer, max_length, activation, precision
        self._act = _native.RERANK_SIGMOID if activation == "sigmoid" else _native.RERANK_IDENTITY
        self._emb = _native.Embedder(engine, config["num_hidden_layers"], config["hidden_size"], config["num_attention_heads"],
                                     config["intermediate_size"], config["vocab_size"], config.get("max_position_embeddings", 512),
                                     config.get("type_vocab_size", 2), config.get("layer_norm_eps", 1e-12))
        self._emb.load_state_dict(state_dict, head=True)
        # "fp16": fp16 GEMM / attention operands, one tensor-core product per step, fp32 accumulation and everything else.  The
        # scores of a query's candidates are only compared with each other, so they need not be held to fp32 arithmetic.
        self._emb.set_precision(precision)
        self._mu = threading.Lock()          # one call at a time: the cross-encoder owns one set of activation buffers

    @classmethod
    def from_pretrained(cls, engine, model_dir: str, **kw):
        """model_dir: a cross-encoder snapshot (config.json, vocab.txt, model.safetensors or pytorch_model.bin,
        tokenizer_config.json when present).  Raises ValueError when it asks for what K5 does not compute."""
        from .text import WordPieceTokenizer
        spec = read_cross_encoder_spec(model_dir)
        cfg = _json(os.path.join(model_dir, "config.json"))
        state = load_state(model_dir)
        where = os.path.join(model_dir, "model.safetensors" if os.path.exists(os.path.join(model_dir, "model.safetensors"))
                             else "pytorch_model.bin")
        check_head_tensors(where, state, cfg["hidden_size"])
        tok = WordPieceTokenizer.from_file(os.path.join(model_dir, "vocab.txt"), do_lower_case=spec["do_lower_case"],
                                           max_length=spec["max_length"])
        kw.setdefault("max_length", spec["max_length"])
        kw.setdefault("activation", spec["activation"])
        return cls(engine, tok, cfg, state, **kw)

    def encode_passages(self, texts: list[str]) -> list[tuple[np.ndarray, int]]:
        """(ids without specials cut at max_length - 3, full length) of each text: what pair truncation needs of a passage"""
        keep = self.max_length - 3
        return [(np.ascontiguousarray(t[:keep]), len(t)) for t in self.tokenizer.encode_batch_plain(texts)]

    def rerank(self, queries: list[str], candidates: list, top_k: int, passages):
        """(positions int32 [n_queries, top_k], scores float32 [n_queries, top_k]) of each query's best top_k candidates
        (position within its candidate list; -1 / NaN past its count), ties by position ascending"""
        qs = [(q, len(q)) for q in self.tokenizer.encode_batch_plain(list(queries))]
        docs = [passages(c, self.encode_passages) for c in candidates]
        flat, toff, seg, poff = build_pairs(self.tokenizer.cls, self.tokenizer.sep, qs, docs, self.max_length)
        with self._mu:
            return self._emb.rerank(poff, flat, toff, seg, top_k, self._act)
