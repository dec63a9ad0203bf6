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


def store_bytes_from_env(colbert: bool) -> int:
    """KRAG_RERANK_STORE_GB (default 0: off): the device bytes (GB = 10^9 bytes) a ColBERT reranker may spend on stored
    passage vectors, over all indexes; a ValueError for a value that is not a number, is negative, or asks a
    cross-encoder to store (its passages are scored with their queries, so there is nothing to store)"""
    raw = os.getenv("KRAG_RERANK_STORE_GB") or "0"
    try:
        gb = float(raw)
    except ValueError:
        raise ValueError(f"KRAG_RERANK_STORE_GB {raw!r}: expected a number of GB") from None
    if not gb >= 0 or gb == float("inf"):
        raise ValueError(f"KRAG_RERANK_STORE_GB {raw!r}: must be a finite number >= 0")
    if gb > 0 and not colbert:
        raise ValueError(f"KRAG_RERANK_STORE_GB {raw!r}: only a ColBERT reranker stores passage vectors (this one is a cross-encoder)")
    return int(gb * 1e9)


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


# ------------------------------------------------------------------ late interaction (ColBERT)
# Stanford ColBERT (colbert.modeling) restated: a query is [CLS] [Q] q... [SEP] cut to query_maxlen and padded with [MASK] to
# exactly query_maxlen (ColBERT tokenises ". " + text and overwrites the "." at position 1 with the marker); a passage is
# [CLS] [D] d... [SEP] cut to doc_maxlen.  Every token row becomes normalize(W h); score = sum over query rows of the max over
# passage rows (skiplist rows excluded) of their dot product.  K5 computes all of it (krag_late_rerank).
COLBERT_QUERY_ROWS = 32          # the longest query_maxlen maxsim_kernel stages


def is_colbert_snapshot(model_dir: str) -> bool:
    """a Stanford ColBERT checkpoint (artifact.metadata, or config.json architectures HF_ColBERT) or a PyLate one (modules.json
    with a Dense module after the Transformer)"""
    join = os.path.join
    if os.path.isfile(join(model_dir, "artifact.metadata")):
        return True
    cfg = _json(join(model_dir, "config.json"), required=False) or {}
    if "HF_ColBERT" in (cfg.get("architectures") or []):
        return True
    mods = _json(join(model_dir, "modules.json"), required=False)
    return isinstance(mods, list) and any(isinstance(m, dict) and str(m.get("type", "")).endswith("Dense") for m in mods)


def _int_field(where: str, meta: dict, field: str, lo: int, hi: int) -> int:
    v = meta.get(field)
    if not isinstance(v, int) or isinstance(v, bool) or not lo <= v <= hi:
        raise ValueError(f"{where}: {field} {v!r}: must be an integer in [{lo}, {hi}]")
    return v


def _marker(where: str, field: str, v, vocab: list[str]) -> int:
    """a marker token given as its vocabulary string ("[unused0]") or its id"""
    if isinstance(v, str) and v in vocab:
        return vocab.index(v)
    if isinstance(v, int) and not isinstance(v, bool) and 0 <= v < len(vocab):
        return v
    raise ValueError(f"{where}: {field} {v!r}: not a token of vocab.txt")


def read_colbert_spec(model_dir: str) -> dict:
    """What Stanford ColBERT computes from a checkpoint, or a ValueError naming the file and field K5 does not restate.
    Reads JSON and vocab.txt only (no weights, no GPU).  Forms:
      Stanford  config.json (a BERT inside K5's shapes) + artifact.metadata (query_maxlen, doc_maxlen, dim,
                mask_punctuation, attend_to_mask_tokens, query_token_id, doc_token_id, similarity); linear.weight in the
                checkpoint's weights
      PyLate    modules.json (Transformer, then a Dense module at `path`), <path>/config.json (out_features, bias false,
                Identity activation), config_sentence_transformers.json (query_prefix, document_prefix, query_length,
                document_length, attend_to_expansion_tokens, skiplist_words, do_query_expansion true) [3P-unverified]
    Stanford's `interaction` must be "colbert" (MaxSim) when present.  Returns query_maxlen, doc_maxlen, dim, attend_to_mask_tokens, q_marker / d_marker (ids), mask_punctuation,
    skip_words (None: string.punctuation), do_lower_case, weight (file, tensor name) of the projection."""
    import string
    join = os.path.join
    cpath = join(model_dir, "config.json")
    cfg = _json(cpath)
    check_bert_config(cpath, cfg)
    vpath = join(model_dir, "vocab.txt")
    if not os.path.isfile(vpath):
        raise ValueError(f"{vpath}: file missing (K5 takes WordPiece vocabularies)")
    with open(vpath, encoding="utf-8") as f:
        vocab = [line.rstrip("\n") for line in f]
    if "[MASK]" not in vocab:
        raise ValueError(f"{vpath}: no [MASK] token (ColBERT pads queries with [MASK])")
    tc = _json(join(model_dir, "tokenizer_config.json"), required=False) or {}
    lower = bool(tc.get("do_lower_case", True))
    max_pos = cfg.get("max_position_embeddings", 512)
    mpath = join(model_dir, "artifact.metadata")
    if os.path.isfile(mpath):
        meta = _json(mpath)
        sim = meta.get("similarity", "cosine")
        if sim != "cosine":
            raise ValueError(f"{mpath}: similarity {sim!r}: K5 scores with ColBERT's cosine MaxSim only")
        inter = meta.get("interaction", "colbert")
        if inter != "colbert":
            raise ValueError(f"{mpath}: interaction {inter!r}: K5 scores with ColBERT's MaxSim interaction only")
        spec = {"query_maxlen": _int_field(mpath, meta, "query_maxlen", 3, COLBERT_QUERY_ROWS),
                "doc_maxlen": _int_field(mpath, meta, "doc_maxlen", 3, max_pos),
                "dim": _int_field(mpath, meta, "dim", 16, 256),
                "q_marker": _marker(mpath, "query_token_id", meta.get("query_token_id", "[unused0]"), vocab),
                "d_marker": _marker(mpath, "doc_token_id", meta.get("doc_token_id", "[unused1]"), vocab),
                "skip_words": None, "do_lower_case": lower}
        for flag, default in (("mask_punctuation", True), ("attend_to_mask_tokens", False)):
            v = meta.get(flag, default)
            if not isinstance(v, bool):
                raise ValueError(f"{mpath}: {flag} {v!r}: must be true or false")
            spec[flag] = v
        if spec["dim"] % 16:
            raise ValueError(f"{mpath}: dim {spec['dim']}: K5 projects to multiples of 16")
        st = join(model_dir, "model.safetensors")
        spec["weight"] = (st if os.path.exists(st) else join(model_dir, "pytorch_model.bin"), "linear.weight")
        return spec
    mods = _json(join(model_dir, "modules.json"), required=False)
    dense = [m for m in (mods or []) if isinstance(m, dict) and str(m.get("type", "")).endswith("Dense")]
    if not dense:
        raise ValueError(f"{mpath}: file missing (a ColBERT snapshot has artifact.metadata, or a PyLate modules.json with a Dense module)")
    if (len(mods) != 2 or len(dense) != 1 or mods[1] is not dense[0]
            or not str(mods[0].get("type", "")).endswith("models.Transformer")):
        raise ValueError(f"{join(model_dir, 'modules.json')}: {[m.get('type') for m in mods]!r}: K5 runs a Transformer followed by one Dense module")
    dpath = join(model_dir, dense[0].get("path", ""), "config.json")
    dc = _json(dpath)
    if dc.get("bias", True):
        raise ValueError(f"{dpath}: bias {dc.get('bias', True)!r}: ColBERT's projection has no bias")
    act = str(dc.get("activation_function", "torch.nn.modules.linear.Identity"))
    if not act.endswith("Identity"):
        raise ValueError(f"{dpath}: activation_function {act!r}: ColBERT's projection is linear")
    if dc.get("in_features") != cfg["hidden_size"]:
        raise ValueError(f"{dpath}: in_features {dc.get('in_features')!r}: config.json hidden_size is {cfg['hidden_size']}")
    spath = join(model_dir, "config_sentence_transformers.json")
    sc = _json(spath)
    if sc.get("do_query_expansion", True) is not True:
        raise ValueError(f"{spath}: do_query_expansion {sc.get('do_query_expansion')!r}: ColBERT pads queries with [MASK]")
    att = sc.get("attend_to_expansion_tokens", False)
    if not isinstance(att, bool):
        raise ValueError(f"{spath}: attend_to_expansion_tokens {att!r}: must be true or false")
    words = sc.get("skiplist_words", list(string.punctuation))
    if not isinstance(words, list) or not all(isinstance(w, str) for w in words):
        raise ValueError(f"{spath}: skiplist_words {words!r}: must be a list of strings")
    spec = {"query_maxlen": _int_field(spath, sc, "query_length", 3, COLBERT_QUERY_ROWS),
            "doc_maxlen": _int_field(spath, sc, "document_length", 3, max_pos),
            "dim": _int_field(dpath, dc, "out_features", 16, 256),
            "q_marker": _marker(spath, "query_prefix", sc.get("query_prefix", "[unused0]"), vocab),
            "d_marker": _marker(spath, "document_prefix", sc.get("document_prefix", "[unused1]"), vocab),
            "mask_punctuation": bool(words), "attend_to_mask_tokens": att, "skip_words": words, "do_lower_case": lower}
    if spec["dim"] % 16:
        raise ValueError(f"{dpath}: out_features {spec['dim']}: K5 projects to multiples of 16")
    wdir = join(model_dir, dense[0].get("path", ""))
    st = join(wdir, "model.safetensors")
    spec["weight"] = (st if os.path.exists(st) else join(wdir, "pytorch_model.bin"), "linear.weight")
    return spec


def colbert_query_ids(tokenizer, texts: list[str], query_maxlen: int, q_marker: int, mask_id: int, attend_to_mask: bool):
    """(ids int32 [n, query_maxlen], key counts int32 [n]): [CLS] [Q] q... [SEP] cut to query_maxlen, [MASK] up to it; the
    keys are the rows before the [MASK] padding, or all rows when attend_to_mask"""
    ids = np.full((len(texts), query_maxlen), mask_id, np.int32)
    keys = np.empty(len(texts), np.int32)
    for i, t in enumerate(tokenizer.encode_batch_plain(list(texts))):
        t = t[:query_maxlen - 3]
        n = len(t) + 3
        ids[i, 0], ids[i, 1], ids[i, 2:n - 1], ids[i, n - 1] = tokenizer.cls, q_marker, t, tokenizer.sep
        keys[i] = query_maxlen if attend_to_mask else n
    return ids, keys


def colbert_skip_ids(tokenizer, words) -> np.ndarray:
    """ColBERT's skiplist as ids: the first token id of each word (string.punctuation's characters by default)"""
    import string
    words = list(string.punctuation) if words is None else list(words)
    return np.unique(np.asarray([t[0] for t in tokenizer.encode_batch_plain(words) if len(t)], np.int32))


def _pack(docs):
    """(tokens, offsets, keep) of encode_passages' output, packed"""
    off = np.zeros(len(docs) + 1, np.int32)
    np.cumsum([len(d[0]) for d in docs], out=off[1:])
    tok = np.concatenate([d[0] for d in docs]) if docs else np.zeros(0, np.int32)
    keep = np.concatenate([d[1] for d in docs]) if docs else np.zeros(0, np.uint8)
    return tok, off, keep


class PassageStore:
    """One index's ColBERT passage vectors on the reranker's GPU (a _native.LateStore, one entry per node ordinal) and the
    host's record of which ordinals it holds: GpuLateInteractionReranker.rerank scores those from the store and encodes the
    others in the call.  Every call holds the reranker's lock (the store works on the embedder's stream and scratch)."""

    APPEND_BATCH = 8192              # passages tokenised and appended per native call (bounds the host's token arrays)

    def __init__(self, reranker: "GpuLateInteractionReranker", native):
        self._rr, self.native = reranker, native
        self.stored = np.zeros(0, bool)

    def __len__(self) -> int:
        return len(self.stored)

    def append(self, texts: list[str]):
        """the next len(texts) ordinals: encode_passages of each text (as rerank() would encode it), stored while the
        budget allows"""
        for i in range(0, len(texts), self.APPEND_BATCH):
            tok, off, keep = _pack(self._rr.encode_passages(texts[i:i + self.APPEND_BATCH]))
            with self._rr._mu:
                got = self.native.append(tok, off, keep)
            self.stored = np.concatenate([self.stored, got.astype(bool)])

    def truncate(self, n: int):
        with self._rr._mu:
            self.native.truncate(n)
        self.stored = self.stored[:n]

    def compact(self, alive):
        """keep the ordinals where alive (bool per ordinal) is set, renumbered in order"""
        alive = np.asarray(alive, bool)
        with self._rr._mu:
            self.native.compact(alive)
        self.stored = self.stored[alive]

    def stats(self) -> dict:
        with self._rr._mu:
            return self.native.stats()

    def destroy(self):
        with self._rr._mu:
            self.native.destroy()


class GpuLateInteractionReranker:
    """A ColBERT late-interaction model on the GPU (krag_late_rerank), with GpuCrossEncoder's interface: rerank(queries,
    candidate ordinals per query, top_k, passages) and encode_passages for the store's per-ordinal token cache.  Each distinct
    candidate ordinal of a call is encoded once.  With store_bytes > 0 (KRAG_RERANK_STORE_GB), create_store gives each index
    a PassageStore, filled at /index, and rerank(..., store=) encodes only the candidates it does not hold."""

    def __init__(self, engine, tokenizer, config: dict, state_dict: dict, weight: np.ndarray, spec: dict, precision: str = "fp32",
                 store_bytes: int = 0):
        from . import _native
        if precision not in PRECISIONS:
            raise ValueError(f"precision {precision!r}: expected 'fp32' or 'fp16'")
        self.tokenizer, self.spec, self.precision = tokenizer, spec, precision
        self.mask_id = tokenizer.vocab["[MASK]"]
        self.skip = colbert_skip_ids(tokenizer, spec["skip_words"]) if spec["mask_punctuation"] else np.zeros(0, np.int32)
        self._emb = _native.Embedder(engine, config["num_hidden_layers"], config["hidden_size"], config["num_attention_heads"],
                                     config["intermediate_size"], config["vocab_size"], config.get("max_position_embeddings", 512),
                                     config.get("type_vocab_size", 2), config.get("layer_norm_eps", 1e-12))
        self._emb.set_late_interaction(weight)
        self._emb.load_state_dict({k: v for k, v in state_dict.items() if k != "linear.weight"})
        self._emb.set_precision(precision)
        self.store_bytes = int(store_bytes)
        if self.store_bytes > 0:
            self._emb.set_store_budget(self.store_bytes)
        self._mu = threading.Lock()

    def create_store(self):
        """a PassageStore for one index, or None when storing is off (store_bytes 0)"""
        if self.store_bytes <= 0:
            return None
        from . import _native
        with self._mu:
            return PassageStore(self, _native.LateStore(self._emb))

    @classmethod
    def from_pretrained(cls, engine, model_dir: str, **kw):
        """model_dir: a ColBERT snapshot (read_colbert_spec); raises ValueError when it asks for what K5 does not compute"""
        from .embedding import _k5_name
        from .text import WordPieceTokenizer
        spec = read_colbert_spec(model_dir)
        cfg = _json(os.path.join(model_dir, "config.json"))
        state = load_state(model_dir)
        wfile, wname = spec["weight"]
        if os.path.dirname(wfile) != model_dir.rstrip(os.sep):          # PyLate: the Dense module's own weights file
            wstate = {_k5_name(k): v for k, v in load_state(os.path.dirname(wfile)).items()}
        else:
            wstate = state
        w = wstate.get(wname)
        if w is None:
            raise ValueError(f"{wfile}: tensor {wname} missing (the ColBERT projection)")
        if tuple(np.shape(w)) != (spec["dim"], cfg["hidden_size"]):
            raise ValueError(f"{wfile}: tensor {wname} has shape {tuple(np.shape(w))}, expected {(spec['dim'], cfg['hidden_size'])}")
        for k in list(wstate):
            if k.startswith("linear.") and k != "linear.weight":
                raise ValueError(f"{wfile}: tensor {k}: ColBERT's projection has no bias")
        tok = WordPieceTokenizer.from_file(os.path.join(model_dir, "vocab.txt"), do_lower_case=spec["do_lower_case"],
                                           max_length=max(spec["doc_maxlen"], spec["query_maxlen"]))
        return cls(engine, tok, cfg, state, np.asarray(w, np.float32), spec, **kw)

    def query_ids(self, texts: list[str]):
        s = self.spec
        return colbert_query_ids(self.tokenizer, texts, s["query_maxlen"], s["q_marker"], self.mask_id, s["attend_to_mask_tokens"])

    def encode_passages(self, texts: list[str]) -> list[tuple[np.ndarray, np.ndarray]]:
        """(ids [CLS] [D] d... [SEP] cut to doc_maxlen, keep mask uint8: 0 on skiplist rows) of each text"""
        keep_n = self.spec["doc_maxlen"] - 3
        out = []
        for t in self.tokenizer.encode_batch_plain(texts):
            ids = np.concatenate([[self.tokenizer.cls, self.spec["d_marker"]], t[:keep_n], [self.tokenizer.sep]]).astype(np.int32)
            out.append((ids, (~np.isin(ids, self.skip)).astype(np.uint8)))
        return out

    def rerank(self, queries: list[str], candidates: list, top_k: int, passages, store: PassageStore | None = None):
        """(positions int32 [n_queries, top_k], scores float32 [n_queries, top_k]) of each query's best top_k candidates
        (position within its candidate list; -1 / NaN past its count), ties by position ascending.  With a store, its
        ordinals are scored from their stored vectors (the same bits) and only the others go through `passages`."""
        q_ids, q_keys = self.query_ids(list(queries))
        poff = np.zeros(len(candidates) + 1, np.int32)
        np.cumsum([len(c) for c in candidates], out=poff[1:])
        flat = np.concatenate([np.asarray(c, np.int64) for c in candidates]) if len(candidates) else np.zeros(0, np.int64)
        uniq, pair_pass = np.unique(flat, return_inverse=True)
        if store is None:
            d_tok, d_off, d_keep = _pack(passages(uniq, self.encode_passages) if len(uniq) else [])
            with self._mu:
                return self._emb.late_rerank(q_ids, q_keys, d_tok, d_off, d_keep, poff, pair_pass.astype(np.int32), top_k)
        held = uniq < len(store.stored)
        held[held] = store.stored[uniq[held]]
        encode = np.flatnonzero(~held)
        source = uniq.astype(np.int32)                    # a stored ordinal names itself, the others ~(position in `encode`)
        source[encode] = ~np.arange(len(encode), dtype=np.int32)
        d_tok, d_off, d_keep = _pack(passages(uniq[encode], self.encode_passages) if len(encode) else [])
        with self._mu:
            return self._emb.late_rerank_stored(store.native, q_ids, q_keys, d_tok, d_off, d_keep, poff, source[pair_pass], top_k)
