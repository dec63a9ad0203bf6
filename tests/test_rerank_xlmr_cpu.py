"""CPU tests of the XLM-RoBERTa reranker path: the Unigram tokenizer (kaito_b200.text.UnigramTokenizer and its native
ASCII path) against the Rust `tokenizers` library on SentencePiece models trained here, pair truncation against the Rust
longest_first rule, and the snapshot reader (read_cross_encoder_spec's xlm-roberta branch) with its refusals."""
import json
import os

import numpy as np
import pytest

from kaito_b200 import _native, text
from kaito_b200.rerank import build_pairs, pair_lengths, read_cross_encoder_spec, xlmr_head_state
from tests import xlmr_reference as xr

FORMS = ["nmt_nfkc", "identity", "legacy", "first"]

FUZZ_FIXED = [
    "", " ", "   ", "hello world", "  leading", "trailing  ", "a  b   c", "tab\tsep\t\tarated", "line\r\nbreak\r\n", "\r\n\r\n", "a\rb\nc",
    "café café CAFÉ CAFÉ", "naïve naïve", "ＦＵＬＬ ｗｉｄｔｈ １２３ ！？", "ﬁle ½ x² ㎏ ℌ", "Ａ́ Ａ́̂",
    "日本語 中文 한국어 各位", "각 한", "москва Привет ЁЖИК", "Ελληνικά العربية हिन्दी",
    "ctl\x00\x01\x07\x1b\x7f end", "\x1c\x1d\x1e\x1f sep", "zero​width‌ joiner‍", "👨‍👩‍👧 family 🏳️‍🌈 flag",
    "﻿bom  nbsp 　ideo  em", "⛄ ☃ ∞ ✓ unknown glyphs 𝔘𝔫𝔦", "x" * 300, "straßeübergrößenträgerin" * 12,
    "<s> literal </s> and <pad><unk><mask>", "x <mask> y", "x  <mask>", "<mask>", " <s>", "＜ｓ＞ full-width specials",
    "the quick brown fox " * 40, "retrieval engine, query: passage?", "``quoted'' text", "email@host.com 3.14 $5",
]


def fuzz_corpus(seed=0, n=600):
    g = np.random.default_rng(seed)
    pool = list("".join(FUZZ_FIXED)) + list(" \t\r\n\x01​́") + ["<s>", "<mask>", "</s>", "  "] + xr.WORDS
    out = list(FUZZ_FIXED) + xr.corpus(seed + 7, 60)
    for _ in range(n):
        out.append("".join(pool[int(i)] for i in g.integers(0, len(pool), int(g.integers(0, 30)))))
    return out


def ascii_corpus(seed=1, n=600):
    g = np.random.default_rng(seed)
    pool = list("abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 .,;:!?'\"`()[]<>/\\-_") + \
        ["\t", "\r\n", "\r", "\n", "\x00", "\x01", "\x0b", "\x0c", "\x1f", "\x7f", "  ", "<s>", "</s>", "<mask>", " <mask>", "<pad>",
         "<unk>", "the", "quick", "brown", "fox", "gpu", "token", "query"]
    out = [t for t in FUZZ_FIXED if t.isascii()]
    for _ in range(n):
        out.append("".join(pool[int(i)] for i in g.integers(0, len(pool), int(g.integers(0, 40)))))
    return out


@pytest.fixture(scope="module")
def tok_paths(tmp_path_factory):
    """tokenizer.json of every form: converted by transformers from a trained nmt_nfkc and identity model, the legacy
    Sequence[Precompiled, Replace] + bare Metaspace form, and that form with prepend_scheme "first" """
    base = tmp_path_factory.mktemp("xlmr_tok")
    nfkc = xr.train_tokenizer(str(base / "nfkc"), seed=0)
    ident = xr.train_tokenizer(str(base / "identity"), seed=1, normalization="identity")
    legacy = xr.legacy_form(os.path.join(nfkc, "tokenizer.json"), str(base / "legacy.json"))
    tj = json.load(open(legacy, encoding="utf-8"))
    tj["pre_tokenizer"]["prepend_scheme"] = "first"
    first = str(base / "first.json")
    json.dump(tj, open(first, "w", encoding="utf-8"), ensure_ascii=False)
    return {"nmt_nfkc": os.path.join(nfkc, "tokenizer.json"), "identity": os.path.join(ident, "tokenizer.json"),
            "legacy": legacy, "first": first, "nfkc_dir": nfkc}


@pytest.mark.parametrize("form", FORMS)
def test_python_ids_match_rust(tok_paths, form):
    from tokenizers import Tokenizer
    ref = Tokenizer.from_file(tok_paths[form])
    tok = text.UnigramTokenizer.from_file(tok_paths[form])
    for s in fuzz_corpus():
        assert tok.encode_py(s) == ref.encode(s, add_special_tokens=False).ids, repr(s)


@pytest.mark.parametrize("form", FORMS)
def test_native_ascii_ids_match_rust(tok_paths, form):
    from tokenizers import Tokenizer
    if not text._native_lib():
        pytest.skip("libkaito_rag.so is not built")
    ref = Tokenizer.from_file(tok_paths[form])
    tok = text.UnigramTokenizer.from_file(tok_paths[form])
    assert tok._nat is not None
    texts = ascii_corpus()
    got = tok.encode_batch_plain(texts)
    for s, g in zip(texts, got):
        assert g.dtype == np.int32 and g.tolist() == ref.encode(s, add_special_tokens=False).ids, repr(s)
    # a mixed batch: ASCII texts natively, the others through Python, in their places
    mixed = fuzz_corpus(3, 50)
    for s, g in zip(mixed, tok.encode_batch_plain(mixed)):
        assert g.tolist() == ref.encode(s, add_special_tokens=False).ids, repr(s)


def test_native_count_past_the_buffer_is_redone(tok_paths):
    """the native encoder reports a text's true count when it exceeds the buffer; the host grows it and asks again"""
    if not text._native_lib():
        pytest.skip("libkaito_rag.so is not built")
    from tokenizers import Tokenizer
    ref = Tokenizer.from_file(tok_paths["nmt_nfkc"])
    tok = text.UnigramTokenizer.from_file(tok_paths["nmt_nfkc"])
    s = "q z " * 50                                   # unknown-heavy: close to one id per character
    assert tok.encode_batch_plain([s, "x"])[0].tolist() == ref.encode(s, add_special_tokens=False).ids


def test_specials_and_surface(tok_paths):
    tok = text.UnigramTokenizer.from_file(tok_paths["nmt_nfkc"], max_length=512)
    assert (tok.cls, tok.sep, tok.max_length) == (0, 2, 512)
    assert tok.encode_batch_plain([]) == []


@pytest.mark.parametrize("max_length", [5, 8, 16, 33, 128, 512])
def test_pairs_match_rust_longest_first(tok_paths, max_length):
    from tokenizers import Tokenizer
    ref = Tokenizer.from_file(tok_paths["nmt_nfkc"])
    ref.enable_truncation(max_length, strategy="longest_first")
    tok = text.UnigramTokenizer.from_file(tok_paths["nmt_nfkc"])
    g = np.random.default_rng(max_length)
    words = xr.WORDS + ["<mask>", "x", "zz"]
    for _ in range(40):
        q = " ".join(g.choice(words, int(g.integers(0, 30))))
        d = " ".join(g.choice(words, int(g.integers(0, 300))))
        qi, di = tok.encode_batch_plain([q, d])
        flat, toff, seg, poff = build_pairs(tok.cls, tok.sep, [(qi, len(qi))], [[(di[:max_length - 3], len(di))]], max_length, 2)
        assert seg is None and toff.tolist() == [0, len(flat)] and poff.tolist() == [0, 1]
        assert flat.tolist() == ref.encode(q, d).ids, (q, d)


def test_pair_lengths_keep_the_bert_rule():
    for nq, nd, m in [(3, 100, 13), (100, 3, 13), (10, 10, 13), (10, 10, 14), (11, 10, 14), (0, 50, 13), (2, 3, 13)]:
        assert pair_lengths(nq, nd, m) == pair_lengths(nq, nd, m, 3) == pair_lengths(nq, nd, m + 1, 4)


# ------------------------------------------------------------------------------------------------ snapshot reader
def _snapshot(path, tok_paths, config=None, tokenizer_config=None, tokenizer_json=None):
    snap = xr.write_snapshot(str(path), config or xr.config_json("bge-reranker-base"), tok_paths["nfkc_dir"], tokenizer_config)
    if tokenizer_json is not None:
        with open(os.path.join(snap, "tokenizer.json"), "w", encoding="utf-8") as f:
            json.dump(tokenizer_json, f, ensure_ascii=False)
    return snap


def test_bge_reranker_snapshots_are_accepted(tmp_path, tok_paths):
    spec = read_cross_encoder_spec(_snapshot(tmp_path / "base", tok_paths))
    assert spec == {"model_type": "xlm-roberta", "max_length": 512, "position_offset": 2, "specials": 4, "activation": "sigmoid"}
    v2 = xr.config_json("bge-reranker-v2-m3")
    spec = read_cross_encoder_spec(_snapshot(tmp_path / "v2", tok_paths, v2, {"model_max_length": 8192}))
    assert spec["max_length"] == 8192 and spec["position_offset"] == 2
    # no limit in tokenizer_config.json: every position row past the offset
    spec = read_cross_encoder_spec(_snapshot(tmp_path / "nolimit", tok_paths, tokenizer_config={"model_max_length": int(1e30)}))
    assert spec["max_length"] == 512
    rob = xr.config_json("bge-reranker-base", model_type="roberta", architectures=["RobertaForSequenceClassification"],
                         sentence_transformers={"activation_fn": "torch.nn.modules.linear.Identity"})
    spec = read_cross_encoder_spec(_snapshot(tmp_path / "roberta", tok_paths, rob))
    assert spec["model_type"] == "roberta" and spec["activation"] == "identity"


def _tj(tok_paths, **model_change):
    tj = json.load(open(tok_paths["nmt_nfkc"], encoding="utf-8"))
    tj["model"].update(model_change)
    return tj


@pytest.mark.parametrize("case,file,field", [
    ("two labels", "config.json", "2 labels"),
    ("BertModel", "config.json", "architectures"),
    ("byte_fallback", "tokenizer.json", "model.byte_fallback"),
    ("BPE", "tokenizer.json", "model.type 'BPE'"),
    ("no tokenizer.json", "tokenizer.json", "file missing"),
    ("model_max_length", "tokenizer_config.json", "model_max_length 513"),
    ("head dim 48", "config.json", "num_attention_heads 16"),
    ("vocab_size", "tokenizer.json", "vocab_size 100"),
    ("normalizer", "tokenizer.json", "normalizer 'NFKC'"),
    ("pre_tokenizer", "tokenizer.json", "pre_tokenizer 'ByteLevel'"),
    ("decoder", "config.json", "is_decoder"),
])
def test_refusals_name_the_file_and_field(tmp_path, tok_paths, case, file, field):
    cfg, tc, tj = xr.config_json("bge-reranker-base"), None, None
    if case == "two labels":
        cfg["id2label"] = {"0": "a", "1": "b"}
    elif case == "BertModel":
        cfg["architectures"] = ["BertModel"]
    elif case == "byte_fallback":
        tj = _tj(tok_paths, byte_fallback=True)
    elif case == "BPE":
        tj = _tj(tok_paths, type="BPE")
    elif case == "model_max_length":
        tc = {"model_max_length": 513}
    elif case == "head dim 48":
        cfg["num_attention_heads"] = 16
    elif case == "vocab_size":
        cfg["vocab_size"] = 100
    elif case == "normalizer":
        tj = _tj(tok_paths)
        tj["normalizer"] = {"type": "NFKC"}
    elif case == "pre_tokenizer":
        tj = _tj(tok_paths)
        tj["pre_tokenizer"] = {"type": "ByteLevel", "add_prefix_space": False}
    elif case == "decoder":
        cfg["is_decoder"] = True
    snap = _snapshot(tmp_path, tok_paths, cfg, tc, tj)
    if case == "no tokenizer.json":
        os.remove(os.path.join(snap, "tokenizer.json"))
    with pytest.raises(ValueError) as e:
        read_cross_encoder_spec(snap)
    assert str(e.value).startswith(os.path.join(snap, file) + ":") and field in str(e.value), str(e.value)


def test_xlmr_embedders_stay_refused(tmp_path, tok_paths):
    """the embedding reader keeps refusing XLM-R: only the cross-encoder reader dispatches on model_type"""
    from kaito_b200.embedding import read_snapshot_spec
    snap = _snapshot(tmp_path, tok_paths)
    with pytest.raises(ValueError, match="model_type 'xlm-roberta'"):
        read_snapshot_spec(snap)


def test_head_mapping():
    st = {"roberta.embeddings.word_embeddings.weight": 1, "roberta.encoder.layer.0.output.dense.bias": 2,
          "roberta.pooler.dense.weight": 3, "classifier.dense.weight": 4, "classifier.dense.bias": 5,
          "classifier.out_proj.weight": 6, "classifier.out_proj.bias": 7}
    assert xlmr_head_state(st) == {"embeddings.word_embeddings.weight": 1, "encoder.layer.0.output.dense.bias": 2,
                                   "pooler.dense.weight": 4, "pooler.dense.bias": 5, "classifier.weight": 6, "classifier.bias": 7}


def test_service_exits_on_a_refused_xlmr_snapshot_before_any_gpu_work(tmp_path, tok_paths, monkeypatch):
    import sys
    from kaito_b200 import service
    monkeypatch.setattr(sys, "setswitchinterval", lambda s: None)

    def no_gpu(*a, **k):
        raise AssertionError("the service reached the GPU")
    monkeypatch.setattr(_native, "Context", no_gpu)
    monkeypatch.delenv("KRAG_MODEL_DIR", raising=False)
    monkeypatch.setenv("EMBEDDING_SOURCE_TYPE", "local")
    monkeypatch.setenv("VECTOR_DB_TYPE", "faiss")
    monkeypatch.delenv("KRAG_RERANK_PRECISION", raising=False)
    snap = _snapshot(tmp_path, tok_paths, tokenizer_json=_tj(tok_paths, byte_fallback=True))
    monkeypatch.setenv("KRAG_RERANK_MODEL_DIR", snap)
    with pytest.raises(SystemExit, match=r"reranker '.*' is not supported by this image: .*tokenizer.json: model.byte_fallback"):
        service.main()


class RecordingEmbedder:
    """the calls GpuCrossEncoder makes on _native.Embedder"""
    made = []

    def __init__(self, *a):
        self.args, self.calls = a, []
        RecordingEmbedder.made.append(self)

    def load_state_dict(self, state, head=False):
        self.calls.append(("load", sorted(k for k in state if k.startswith(("pooler.", "classifier."))), head))

    def set_precision(self, precision):
        self.calls.append(("precision", precision))

    def set_position_offset(self, off):
        self.calls.append(("offset", off))

    def rerank(self, poff, flat, toff, seg, top_k, act):
        self.calls.append(("rerank", flat.tolist(), toff.tolist(), seg, top_k))
        return np.zeros((len(poff) - 1, top_k), np.int32), np.zeros((len(poff) - 1, top_k), np.float32)


def test_from_pretrained_wires_the_xlmr_spec(tmp_path, tok_paths, monkeypatch):
    from kaito_b200.rerank import GpuCrossEncoder
    monkeypatch.setattr(_native, "Embedder", RecordingEmbedder)
    d = 768
    state = {"roberta.embeddings.word_embeddings.weight": np.zeros((4, d), np.float32),
             "classifier.dense.weight": np.zeros((d, d), np.float32), "classifier.dense.bias": np.zeros(d, np.float32),
             "classifier.out_proj.weight": np.zeros((1, d), np.float32), "classifier.out_proj.bias": np.zeros(1, np.float32)}
    snap = _snapshot(tmp_path, tok_paths)
    from safetensors.numpy import save_file
    save_file(state, os.path.join(snap, "model.safetensors"))
    ce = GpuCrossEncoder.from_pretrained(None, snap, precision="fp16")
    e = RecordingEmbedder.made[-1]
    assert e.args[1:] == (12, 768, 12, 3072, xr.VOCAB, 514, 1, 1e-5)
    assert e.calls == [("load", ["classifier.bias", "classifier.weight", "pooler.dense.bias", "pooler.dense.weight"], True),
                       ("precision", "fp16"), ("offset", 2)]
    assert ce.max_length == 512 and ce.specials == 4 and isinstance(ce.tokenizer, text.UnigramTokenizer)
    ce.rerank(["gpu token"], [[0]], 1, lambda ords, enc: enc(["the quick fox"]))
    _, flat, toff, seg, top_k = e.calls[-1]
    q, dd = ce.tokenizer.encode_batch_plain(["gpu token", "the quick fox"])
    assert flat == [0] + q.tolist() + [2, 2] + dd.tolist() + [2] and toff == [0, len(flat)] and seg is None and top_k == 1
