"""Cross-encoder reranking of /retrieve candidates: a BERT cross-encoder (BertForSequenceClassification with one label, e.g.
cross-encoder/ms-marco-MiniLM-L-6-v2) or an XLM-RoBERTa one (XLMRobertaForSequenceClassification with one label, e.g.
BAAI/bge-reranker-base / -large / -v2-m3) scores each (query, passage) pair on the GPU -- the K5 encoder (token types for
BERT's second segment, positions from pad_token_id + 1 for XLM-R), the pooler and classifier head, and a per-query top-k
selection, all in libkaito_rag (kaito_b200/csrc/embed.cu).
The hybrid stage hands over N = min(max(top_k, KRAG_RERANK_CANDIDATES), RAG_MAX_TOP_K) fused candidates per query and the
reranker keeps the top_k best (LlamaIndex's retriever similarity_top_k, then the postprocessor's top_n)."""
from __future__ import annotations

import os
import threading

import numpy as np

from .embedding import _json, check_bert_config, load_state
from .text import read_unigram_json

RERANK_CANDIDATES = 30           # KRAG_RERANK_CANDIDATES default
_ACTIVATIONS = {"Sigmoid": "sigmoid", "Identity": "identity"}
_XLMR_TYPES = {"xlm-roberta": "XLMRobertaForSequenceClassification", "roberta": "RobertaForSequenceClassification"}
PRECISIONS = ("fp32", "fp16")    # KRAG_RERANK_PRECISION; the default is the fp32-accurate forward


def precision_from_env() -> str:
    """KRAG_RERANK_PRECISION: "fp32" (default) or "fp16"; a ValueError for anything else"""
    p = os.getenv("KRAG_RERANK_PRECISION") or "fp32"
    if p not in PRECISIONS:
        raise ValueError(f"KRAG_RERANK_PRECISION {p!r}: expected 'fp32' or 'fp16'")
    return p


def _activation(cpath: str, cfg: dict) -> str:
    st = cfg.get("sentence_transformers") if isinstance(cfg.get("sentence_transformers"), dict) else {}
    fn = st.get("activation_fn") or cfg.get("sbert_ce_default_activation_function") or "torch.nn.modules.activation.Sigmoid"
    act = _ACTIVATIONS.get(str(fn).rsplit(".", 1)[-1]) if isinstance(fn, str) and fn.startswith("torch.nn.") else None
    if act is None:
        raise ValueError(f"{cpath}: activation function {fn!r}: K5 applies torch.nn Sigmoid or Identity only")
    return act


def _one_label(cpath: str, cfg: dict):
    labels = len(cfg["id2label"]) if isinstance(cfg.get("id2label"), dict) else cfg.get("num_labels", 2)
    if labels != 1:
        raise ValueError(f"{cpath}: {labels} labels (num_labels / id2label): K5 reranks with one relevance logit only")


def read_cross_encoder_spec(model_dir: str) -> dict:
    """What sentence-transformers' CrossEncoder computes from a snapshot, or a ValueError naming the file and field that asks
    for something K5 does not compute.  Reads JSON only (no weights, no GPU).  config.json model_type "xlm-roberta" or
    "roberta" is read by read_xlmr_cross_encoder_spec; every other snapshot as a BERT cross-encoder, which returns
      max_length     tokens per pair incl. [CLS] / [SEP] / [SEP]: tokenizer_config.json model_max_length, else
                     config.json max_position_embeddings (default 512); a limit beyond the position table is refused
      do_lower_case  tokenizer_config.json do_lower_case (default true)
      activation     "sigmoid" | "identity": config.json sentence_transformers.activation_fn or the legacy
                     sbert_ce_default_activation_function; Sigmoid when neither is given (the default for one label)
                     [3P-unverified]"""
    join = os.path.join
    cpath = join(model_dir, "config.json")
    cfg = _json(cpath)
    if cfg.get("model_type") in _XLMR_TYPES:
        return read_xlmr_cross_encoder_spec(model_dir, cfg)
    check_bert_config(cpath, cfg)
    archs = cfg.get("architectures") or []
    if "BertForSequenceClassification" not in archs:
        raise ValueError(f"{cpath}: architectures {archs!r}: a cross-encoder is a BertForSequenceClassification")
    _one_label(cpath, cfg)
    if not isinstance(cfg.get("type_vocab_size", 2), int) or cfg.get("type_vocab_size", 2) < 2:
        raise ValueError(f"{cpath}: type_vocab_size {cfg.get('type_vocab_size')!r}: sentence pairs need token type 1")
    act = _activation(cpath, cfg)
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


def read_xlmr_cross_encoder_spec(model_dir: str, cfg: dict) -> dict:
    """The XLM-RoBERTa branch of read_cross_encoder_spec (bge-reranker-base / -large / -v2-m3): an encoder K5 runs as a BERT
    with positions from pad_token_id + 1 and one token-type row, pairs <s> q </s></s> d </s>, and the classification head
    dense -> tanh -> out_proj on the <s> row (BERT's pooler and classifier).  Returns
      model_type       "xlm-roberta" | "roberta"
      max_length       tokens per pair incl. its four specials: tokenizer_config.json model_max_length, else
                       max_position_embeddings - pad_token_id - 1 (the rows past the offset)
      position_offset  pad_token_id + 1
      specials         4
      activation       as for BERT: no sentence_transformers key means Sigmoid [3P-unverified]"""
    join = os.path.join
    cpath = join(model_dir, "config.json")
    check_bert_config(cpath, dict(cfg, model_type="bert"))     # the shape rules; model_type was dispatched on
    mt = cfg["model_type"]
    archs = cfg.get("architectures") or []
    if _XLMR_TYPES[mt] not in archs:
        raise ValueError(f"{cpath}: architectures {archs!r}: a {mt} cross-encoder is a {_XLMR_TYPES[mt]}")
    _one_label(cpath, cfg)
    tv = cfg.get("type_vocab_size", 1)
    if not isinstance(tv, int) or tv < 1:
        raise ValueError(f"{cpath}: type_vocab_size {tv!r}: the pairs take token type row 0")
    act = _activation(cpath, cfg)
    pad = cfg.get("pad_token_id", 1)
    max_pos = cfg.get("max_position_embeddings", 514)
    if not isinstance(pad, int) or pad < 0 or not isinstance(max_pos, int) or max_pos - pad - 1 < 4:
        raise ValueError(f"{cpath}: pad_token_id {pad!r}, max_position_embeddings {max_pos!r}: positions start at "
                         "pad_token_id + 1 and a pair needs at least 4 of them")
    limit = max_pos - pad - 1
    tpath = join(model_dir, "tokenizer_config.json")
    tc = _json(tpath, required=False) or {}
    mml = tc.get("model_max_length")
    if isinstance(mml, (int, float)) and not isinstance(mml, bool) and mml >= 1e12:
        mml = None                           # transformers' "no limit" sentinel (int(1e30))
    max_length = limit if mml is None else mml
    if not isinstance(max_length, int) or not 4 <= max_length <= limit:
        raise ValueError(f"{tpath}: model_max_length {max_length!r}: must be an integer in [4, config.json "
                         f"max_position_embeddings {max_pos} - pad_token_id {pad} - 1 = {limit}]")
    jpath = join(model_dir, "tokenizer.json")
    if not os.path.isfile(jpath):
        raise ValueError(f"{jpath}: file missing (XLM-R rerankers are read with their SentencePiece Unigram tokenizer.json)")
    tj = read_unigram_json(jpath)
    n_ids = max([len(tj["pieces"])] + [i + 1 for _, i, _, _ in tj["added"]])
    if n_ids > cfg.get("vocab_size", 0):
        raise ValueError(f"{jpath}: model.vocab / added_tokens: {n_ids} ids, more than config.json vocab_size "
                         f"{cfg.get('vocab_size')!r} (K5 clamps ids to the word table, it does not reject them)")
    return {"model_type": mt, "max_length": max_length, "position_offset": pad + 1, "specials": 4, "activation": act}


def check_head_tensors(where: str, state: dict, hidden: int):
    """the classifier head a one-label BertForSequenceClassification carries (names without "bert."), or a ValueError
    naming the file and tensor"""
    for name, shape in (("pooler.dense.weight", (hidden, hidden)), ("pooler.dense.bias", (hidden,)),
                        ("classifier.weight", (1, hidden)), ("classifier.bias", (1,))):
        if name not in state:
            raise ValueError(f"{where}: tensor {name} missing (a cross-encoder carries the pooler and a one-label classifier)")
        if tuple(np.shape(state[name])) != shape:
            raise ValueError(f"{where}: tensor {name} has shape {tuple(np.shape(state[name]))}, expected {shape}")


def pair_lengths(n_q: int, n_d: int, max_length: int, specials: int = 3) -> tuple[int, int]:
    """tokens kept of each half of [CLS] q [SEP] d [SEP] (specials = 3; XLM-R's <s> q </s></s> d </s>: 4) under
    truncation="longest_first" to max_length: the rule of the Rust tokenizers' pair truncation over max_length - specials
    (the shorter half stays whole when it fits in half the budget, else the budget is halved; on equal lengths the first
    half gets the smaller share) [3P-unverified]"""
    budget = max_length - specials
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
                max_length: int, seps: int = 1):
    """packed pairs for krag_rerank: queries[i] = (ids, full length), passages[i] = that query's candidates as (ids cut at
    max_length - 3, full length); seps = the separator run between the halves ([SEP]: 1; XLM-R's </s></s>: 2).  Returns
    (flat int32 ids, token offsets [n_pairs + 1], seg_b [n_pairs] (None when seps = 2: XLM-R pairs are unsegmented), pair
    offsets [n_queries + 1])"""
    parts, lens, seg = [], [], []
    poff = np.zeros(len(queries) + 1, np.int32)
    head, mid, tail = np.asarray([cls_id], np.int32), np.full(seps, sep_id, np.int32), np.asarray([sep_id], np.int32)
    for i, ((q, nq), cands) in enumerate(zip(queries, passages)):
        for d, nd in cands:
            a, b = pair_lengths(nq, nd, max_length, 2 + seps)
            parts += [head, q[:a], mid, d[:b], tail]
            lens.append(a + b + 2 + seps)
            seg.append(a + 1 + seps)
        poff[i + 1] = poff[i] + len(cands)
    toff = np.zeros(len(lens) + 1, np.int32)
    np.cumsum(lens, out=toff[1:])
    flat = np.concatenate(parts).astype(np.int32) if parts else np.zeros(0, np.int32)
    return flat, toff, (np.asarray(seg, np.int32) if seps == 1 else None), poff


def xlmr_head_state(state: dict) -> dict:
    """an XLMRobertaForSequenceClassification state under the names K5 loads: "roberta." stripped, classifier.dense.* as
    pooler.dense.* and classifier.out_proj.* as classifier.* (dense -> tanh -> out_proj on the <s> row is BERT's pooler and
    classifier); a stray pooler of the base model is dropped"""
    out = {}
    for k, v in state.items():
        k = k[8:] if k.startswith("roberta.") else k
        if k.startswith("pooler."):
            continue
        if k.startswith("classifier.dense."):
            k = "pooler.dense." + k[len("classifier.dense."):]
        elif k.startswith("classifier.out_proj."):
            k = "classifier." + k[len("classifier.out_proj."):]
        out[k] = v
    return out


class GpuCrossEncoder:
    """A BERT or XLM-RoBERTa cross-encoder on the GPU (krag_rerank).  rerank(queries, candidate ordinals per query, top_k, passages) scores
    every (query, passage) pair and returns the positions and scores of each query's top_k; `passages(ordinals, encode)` is the
    store's per-ordinal token cache (_IndexState.pair_passages), filled through `encode_passages` on a miss."""

    def __init__(self, engine, tokenizer, config: dict, state_dict: dict, max_length: int = 512, activation: str = "sigmoid",
                 precision: str = "fp32", position_offset: int = 0, specials: int = 3):
        """specials: 3 for [CLS] q [SEP] d [SEP] (token type 1 from d on), 4 for XLM-R's unsegmented <s> q </s></s> d </s>;
        position_offset: the position row of a pair's first token (XLM-R: pad_token_id + 1)"""
        from . import _native
        if activation not in ("sigmoid", "identity"):
            raise ValueError(f"activation {activation!r}: expected 'sigmoid' or 'identity'")
        if precision not in PRECISIONS:
            raise ValueError(f"precision {precision!r}: expected 'fp32' or 'fp16'")
        if specials not in (3, 4):
            raise ValueError(f"specials {specials!r}: expected 3 ([SEP]) or 4 (</s></s>)")
        self.tokenizer, self.max_length, self.activation, self.precision = tokenizer, max_length, activation, precision
        self.specials = specials
        self._act = _native.RERANK_SIGMOID if activation == "sigmoid" else _native.RERANK_IDENTITY
        self._emb = _native.Embedder(engine, config["num_hidden_layers"], config["hidden_size"], config["num_attention_heads"],
                                     config["intermediate_size"], config["vocab_size"], config.get("max_position_embeddings", 512),
                                     config.get("type_vocab_size", 2), config.get("layer_norm_eps", 1e-12))
        self._emb.load_state_dict(state_dict, head=True)
        # "fp16": fp16 GEMM / attention operands, one tensor-core product per step, fp32 accumulation and everything else.  The
        # scores of a query's candidates are only compared with each other, so they need not be held to fp32 arithmetic.
        self._emb.set_precision(precision)
        if position_offset:
            self._emb.set_position_offset(position_offset)
        self._mu = threading.Lock()          # one call at a time: the cross-encoder owns one set of activation buffers

    @classmethod
    def from_pretrained(cls, engine, model_dir: str, **kw):
        """model_dir: a cross-encoder snapshot (config.json, model.safetensors or pytorch_model.bin, tokenizer_config.json
        when present; vocab.txt for BERT, tokenizer.json for XLM-R).  Raises ValueError when it asks for what K5 does not
        compute."""
        from .text import UnigramTokenizer, WordPieceTokenizer
        spec = read_cross_encoder_spec(model_dir)
        cfg = _json(os.path.join(model_dir, "config.json"))
        state = load_state(model_dir)
        where = os.path.join(model_dir, "model.safetensors" if os.path.exists(os.path.join(model_dir, "model.safetensors"))
                             else "pytorch_model.bin")
        if "position_offset" in spec:        # XLM-R
            state = xlmr_head_state(state)
            check_head_tensors(where, state, cfg["hidden_size"])
            tok = UnigramTokenizer.from_file(os.path.join(model_dir, "tokenizer.json"), max_length=spec["max_length"])
            kw.setdefault("position_offset", spec["position_offset"])
            kw.setdefault("specials", spec["specials"])
            cfg = dict(cfg, type_vocab_size=cfg.get("type_vocab_size", 1), max_position_embeddings=cfg.get("max_position_embeddings", 514))
        else:
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
        flat, toff, seg, poff = build_pairs(self.tokenizer.cls, self.tokenizer.sep, qs, docs, self.max_length, self.specials - 2)
        with self._mu:
            return self._emb.rerank(poff, flat, toff, seg, top_k, self._act)
