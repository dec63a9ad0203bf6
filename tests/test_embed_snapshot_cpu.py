"""read_snapshot_spec without a GPU: what a sentence-transformers snapshot asks of K5 (pooling, token budget, casing, query
instruction), the refusal of every snapshot K5 does not compute, each naming its file, and the WordPiece tokenizer built from
the spec against transformers.BertTokenizer on the same vocab.txt."""
import os

import pytest

from kaito_b200.embedding import BGE_QUERY_INSTRUCTION, GpuBertEmbedding, read_snapshot_spec
from kaito_b200.text import WordPieceTokenizer
from tests import st_snapshot as sn


def _spec(tmp_path, kind="bge", **edits):
    """spec of a `kind` snapshot with files replaced (name=content) or removed (name=None); "_json" in a name stands for
    ".json\""""
    files = sn.layout(kind)
    for k, v in edits.items():
        files[k.replace("_json", ".json")] = v
    return read_snapshot_spec(sn.write(tmp_path / "snap", files))


def test_bge_small_layout(tmp_path):
    assert _spec(tmp_path) == {"pooling": "cls", "max_length": 512, "do_lower_case": True,
                               "query_instruction": BGE_QUERY_INSTRUCTION}


def test_all_minilm_layout(tmp_path):
    assert _spec(tmp_path, "minilm") == {"pooling": "mean", "max_length": 256, "do_lower_case": True, "query_instruction": None}


def test_no_modules_json_is_cls(tmp_path):
    """a plain Hugging Face snapshot (no sentence-transformers files) keeps the CLS pooling and the bge prefix"""
    spec = _spec(tmp_path, "minilm", modules_json=None, **{"1_Pooling/config.json": None}, sentence_bert_config_json=None,
                 tokenizer_config_json=None)
    assert spec == {"pooling": "cls", "max_length": 512, "do_lower_case": True, "query_instruction": BGE_QUERY_INSTRUCTION}


def test_normalize_module_is_optional(tmp_path):
    files = sn.layout("minilm")
    files["modules.json"] = files["modules.json"][:2]
    assert read_snapshot_spec(sn.write(tmp_path / "s", files))["pooling"] == "mean"


@pytest.mark.parametrize("tok,cfg_pos,want", [(256, 512, 256), (None, 512, 512), (10 ** 30, 512, 512), (512, 128, 128),
                                             (None, None, 512)])
def test_max_length_without_max_seq_length(tmp_path, tok, cfg_pos, want):
    """sentence-transformers' Transformer: min(tokenizer model_max_length, config max_position_embeddings), 512 without both"""
    files = sn.layout("minilm")
    files["sentence_bert_config.json"] = {"do_lower_case": False}
    if tok is None:
        del files["tokenizer_config.json"]["model_max_length"]
    else:
        files["tokenizer_config.json"]["model_max_length"] = tok
    if cfg_pos is None:
        del files["config.json"]["max_position_embeddings"]
    else:
        files["config.json"]["max_position_embeddings"] = cfg_pos
    assert read_snapshot_spec(sn.write(tmp_path / "s", files))["max_length"] == want


def test_cased_tokenizer(tmp_path):
    files = sn.layout("minilm")
    files["tokenizer_config.json"]["do_lower_case"] = False
    assert read_snapshot_spec(sn.write(tmp_path / "s", files))["do_lower_case"] is False


# ------------------------------------------------------------------------------------------------------------ refusals
def _modules(*types):
    paths = {"Transformer": "", "Pooling": "1_Pooling", "Normalize": "2_Normalize", "Dense": "2_Dense"}
    return [{"idx": i, "name": str(i), "path": paths.get(t, t), "type": "sentence_transformers.models." + t} for i, t in enumerate(types)]


def _pool(**flags):
    return dict(sn.pooling_config(384, "none"), **flags)


REFUSALS = [
    # modules.json: a Transformer, then a Pooling, then an optional Normalize
    ("dense head", dict(modules_json=_modules("Transformer", "Pooling", "Dense", "Normalize")), "modules.json"),
    ("pooling first", dict(modules_json=_modules("Pooling", "Transformer")), "modules.json"),
    ("no pooling", dict(modules_json=_modules("Transformer", "Normalize")), "modules.json"),
    ("two normalize", dict(modules_json=_modules("Transformer", "Pooling", "Normalize", "Normalize")), "modules.json"),
    ("transformer in a subdirectory", dict(modules_json=[dict(_modules("Transformer")[0], path="0_BERT")] +
                                          _modules("Transformer", "Pooling")[1:]), "modules.json"),
    # <pooling path>/config.json: exactly one of cls / mean
    ("max pooling", {"1_Pooling/config.json": _pool(pooling_mode_max_tokens=True)}, "1_Pooling/config.json"),
    ("mean sqrt len", {"1_Pooling/config.json": _pool(pooling_mode_mean_sqrt_len_tokens=True)}, "1_Pooling/config.json"),
    ("weighted mean", {"1_Pooling/config.json": _pool(pooling_mode_weightedmean_tokens=True)}, "1_Pooling/config.json"),
    ("last token", {"1_Pooling/config.json": _pool(pooling_mode_lasttoken=True)}, "1_Pooling/config.json"),
    ("cls + mean", {"1_Pooling/config.json": _pool(pooling_mode_cls_token=True, pooling_mode_mean_tokens=True)},
     "1_Pooling/config.json"),
    ("mean + max", {"1_Pooling/config.json": _pool(pooling_mode_mean_tokens=True, pooling_mode_max_tokens=True)},
     "1_Pooling/config.json"),
    ("no mode", {"1_Pooling/config.json": _pool()}, "1_Pooling/config.json"),
    ("include_prompt false", {"1_Pooling/config.json": _pool(pooling_mode_mean_tokens=True, include_prompt=False)},
     "1_Pooling/config.json"),
    ("pooling width", {"1_Pooling/config.json": dict(sn.pooling_config(768, "mean_tokens"))}, "1_Pooling/config.json"),
    ("pooling config missing", {"1_Pooling/config.json": None}, "1_Pooling/config.json"),
    # sentence_bert_config.json
    ("lower-casing a cased tokenizer", dict(sentence_bert_config_json={"max_seq_length": 256, "do_lower_case": True},
                                            tokenizer_config_json={"do_lower_case": False}), "sentence_bert_config.json"),
    ("longer than the positions", dict(sentence_bert_config_json={"max_seq_length": 1024}), "sentence_bert_config.json"),
    # config.json: what K5 computes
    ("xlm-roberta", dict(config_json=dict(sn.MINILM_L6, model_type="xlm-roberta")), "config.json"),
    ("mpnet", dict(config_json=dict(sn.MINILM_L6, model_type="mpnet")), "config.json"),
    ("distilbert", dict(config_json=dict(sn.MINILM_L6, model_type="distilbert")), "config.json"),
    ("nomic", dict(config_json=dict(sn.MINILM_L6, model_type="nomic_bert")), "config.json"),
    ("relative positions", dict(config_json=dict(sn.MINILM_L6, position_embedding_type="relative_key_query")), "config.json"),
    ("gelu_new", dict(config_json=dict(sn.MINILM_L6, hidden_act="gelu_new")), "config.json"),
    ("relu", dict(config_json=dict(sn.MINILM_L6, hidden_act="relu")), "config.json"),
    ("decoder", dict(config_json=dict(sn.MINILM_L6, is_decoder=True)), "config.json"),
    ("head dim 48", dict(config_json=dict(sn.MINILM_L6, hidden_size=768, num_attention_heads=16)), "config.json"),
    ("head dim 128", dict(config_json=dict(sn.MINILM_L6, hidden_size=1024, num_attention_heads=8)), "config.json"),
    ("hidden 320", dict(config_json=dict(sn.MINILM_L6, hidden_size=320, num_attention_heads=10)), "config.json"),
    ("hidden 1280", dict(config_json=dict(sn.MINILM_L6, hidden_size=1280, num_attention_heads=20)), "config.json"),
    ("intermediate 1000", dict(config_json=dict(sn.MINILM_L6, intermediate_size=1000)), "config.json"),
]


@pytest.mark.parametrize("label,edits,file", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals_name_their_file(tmp_path, label, edits, file):
    with pytest.raises(ValueError) as e:
        _spec(tmp_path, "minilm", **edits)
    assert os.path.join(str(tmp_path / "snap"), file) in str(e.value), str(e.value)


def test_missing_vocab_is_refused(tmp_path):
    with pytest.raises(ValueError, match="vocab.txt"):
        read_snapshot_spec(sn.write(tmp_path / "s", sn.layout("minilm"), vocab=None))


def test_from_pretrained_refuses_before_reading_weights(tmp_path):
    """the refusal comes from the snapshot's JSON files: the weights (here not a safetensors file at all) are never opened
    and no GPU is touched (there is no engine)"""
    files = sn.layout("minilm")
    files["modules.json"] = _modules("Transformer", "Pooling", "Dense")
    d = sn.write(tmp_path / "s", files)
    with open(os.path.join(d, "model.safetensors"), "wb") as f:
        f.write(b"not weights")
    with pytest.raises(ValueError, match="modules.json"):
        GpuBertEmbedding.from_pretrained(None, d)


def test_service_exits_on_a_refused_snapshot(tmp_path, monkeypatch):
    """service.main turns the refusal into the SystemExit every other start-up error gives, before any GPU work"""
    import sys
    from kaito_b200 import service
    monkeypatch.setattr(sys, "setswitchinterval", lambda s: None)
    files = sn.layout("minilm")
    files["config.json"] = dict(sn.MINILM_L6, model_type="mpnet")
    monkeypatch.setenv("KRAG_MODEL_DIR", sn.write(tmp_path / "s", files))
    monkeypatch.setenv("EMBEDDING_SOURCE_TYPE", "local")
    monkeypatch.setenv("VECTOR_DB_TYPE", "faiss")
    with pytest.raises(SystemExit, match="config.json: model_type 'mpnet'"):
        service.main()


# ---------------------------------------------------------------------------------------------- tokenizer from the spec
TEXTS = ["The quick brown Fox jumps over the lazy dog.", "Café naïvely, CAFE cafe café", "中文 日本語 token GPU", "Über über ü Ü é E e",
         "the " * 400, "Fox " * 300 + "中文 " * 100, "re-present this question: a b c abc cab", "", "x" * 120 + " naïve"]


@pytest.mark.parametrize("lower", [True, False])
def test_tokenizer_from_spec_matches_bert_tokenizer(tmp_path, lower):
    transformers = pytest.importorskip("transformers")
    files = sn.layout("minilm")
    files["tokenizer_config.json"]["do_lower_case"] = lower
    d = sn.write(tmp_path / "s", files)
    spec = read_snapshot_spec(d)
    assert spec["do_lower_case"] is lower and spec["max_length"] == 256
    mine = WordPieceTokenizer.from_file(os.path.join(d, "vocab.txt"), do_lower_case=spec["do_lower_case"], max_length=spec["max_length"])
    ref = transformers.BertTokenizer(os.path.join(d, "vocab.txt"), do_lower_case=lower)
    want = [ref.encode(t, add_special_tokens=True, truncation=True, max_length=256) for t in TEXTS]
    assert max(len(w) for w in want) == 256
    for t, w in zip(TEXTS, want):
        assert mine.encode(t) == w, repr(t)
        assert mine.encode_py(t) == w, repr(t)
    flat, offs = mine.encode_batch_flat(TEXTS)
    assert [flat[offs[i]:offs[i + 1]].tolist() for i in range(len(TEXTS))] == want
    if not lower:                                    # casing really reaches the ids
        assert mine.encode("The")[1] != mine.encode("the")[1]
