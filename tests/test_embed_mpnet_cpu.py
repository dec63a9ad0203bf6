"""MPNet sentence embedders (all-mpnet-base-v2, multi-qa-mpnet-base-*) without a GPU: the relative-position bucket K5's
attention applies against transformers' MPNetEncoder.relative_position_bucket, read_snapshot_spec on MPNet-laid-out
snapshots and its refusals (each naming its file), the MPNetModel -> K5 tensor names, and the WordPiece tokenizer with
MPNet's specials against transformers.MPNetTokenizer on the same vocab.txt."""
import os

import numpy as np
import pytest

from kaito_b200 import embedding as E
from kaito_b200.embedding import read_snapshot_spec
from kaito_b200.text import WordPieceTokenizer
from tests import st_snapshot as sn

# config.json of sentence-transformers/all-mpnet-base-v2 (no checkpoint offline: the layouts are restated here)
MPNET_BASE = dict(architectures=["MPNetForMaskedLM"], attention_probs_dropout_prob=0.1, bos_token_id=0, eos_token_id=2,
                  hidden_act="gelu", hidden_dropout_prob=0.1, hidden_size=768, initializer_range=0.02, intermediate_size=3072,
                  layer_norm_eps=1e-05, max_position_embeddings=514, model_type="mpnet", num_attention_heads=12,
                  num_hidden_layers=12, pad_token_id=1, relative_attention_num_buckets=32, vocab_size=30527)
# MPNet vocab.txt: <s> <pad> </s> <unk> first, <mask> last, the BERT vocabulary between
VOCAB = ["<s>", "<pad>", "</s>", "<unk>"] + sn.VOCAB + ["<mask>"]
SPECIALS = {"cls_token": "<s>", "sep_token": "</s>", "unk_token": "[UNK]"}


def mpnet_layout(kind="all-mpnet", config=None):
    """{file name: JSON content} of an all-mpnet-base-v2 ("all-mpnet": mean pooling, Normalize, 384 tokens) or
    multi-qa-mpnet-base-dot-v1 ("multi-qa-dot": CLS pooling, no Normalize, 512 tokens) snapshot"""
    cfg = dict(config or MPNET_BASE)
    cls = kind == "multi-qa-dot"
    modules = [{"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
               {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"}]
    if not cls:
        modules.append({"idx": 2, "name": "2", "path": "2_Normalize", "type": "sentence_transformers.models.Normalize"})
    return {
        "config.json": cfg,
        "tokenizer_config.json": {"bos_token": "<s>", "cls_token": "<s>", "do_lower_case": True, "eos_token": "</s>",
                                  "mask_token": "<mask>", "model_max_length": 512, "pad_token": "<pad>", "sep_token": "</s>",
                                  "strip_accents": None, "tokenize_chinese_chars": True, "tokenizer_class": "MPNetTokenizer",
                                  "unk_token": "[UNK]"},
        "sentence_bert_config.json": {"max_seq_length": 512 if cls else 384, "do_lower_case": False},
        "modules.json": modules,
        "1_Pooling/config.json": sn.pooling_config(cfg["hidden_size"], "cls_token" if cls else "mean_tokens"),
    }


def _write(tmp_path, files, vocab=VOCAB, name="snap"):
    return sn.write(tmp_path / name, files, vocab=vocab)


# ------------------------------------------------------------------------------------------------ relative buckets
def test_relative_bucket_matches_transformers():
    """the bucket the kernel applies (distance clamped to +-128 first) is transformers' for every distance up to 8193"""
    torch = pytest.importorskip("torch")
    from transformers.models.mpnet.modeling_mpnet import MPNetEncoder
    from kaito_b200 import _native
    rel = np.arange(-8193, 8194)
    want = MPNetEncoder.relative_position_bucket(torch.from_numpy(rel), num_buckets=32, max_distance=128).numpy()
    got = np.array([_native.debug_relative_bucket(int(r)) for r in rel])
    assert np.array_equal(got, want), rel[got != want][:10]
    assert set(got.tolist()) == set(range(32)) - {16}    # every row of the table but 16 (a future key at distance 0) is reachable
    assert got[rel == 1][0] == 17 and got[rel == -1][0] == 1 and got[rel == 0][0] == 0   # future keys take the upper half


# ------------------------------------------------------------------------------------------------ snapshot spec
def test_all_mpnet_base_v2_layout(tmp_path):
    assert read_snapshot_spec(_write(tmp_path, mpnet_layout())) == dict(
        {"pooling": "mean", "max_length": 384, "do_lower_case": True, "query_instruction": None, "model_type": "mpnet",
         "position_offset": 2}, **SPECIALS)


def test_multi_qa_mpnet_dot_layout(tmp_path):
    """CLS pooling, no Normalize module, 512 tokens (514 positions - 2), and no bge instruction"""
    assert read_snapshot_spec(_write(tmp_path, mpnet_layout("multi-qa-dot"))) == dict(
        {"pooling": "cls", "max_length": 512, "do_lower_case": True, "query_instruction": None, "model_type": "mpnet",
         "position_offset": 2}, **SPECIALS)


def test_added_token_dict_specials(tmp_path):
    """tokenizer_config.json may state a special as an AddedToken dict; a missing field takes MPNetTokenizer's default"""
    files = mpnet_layout()
    tc = files["tokenizer_config.json"]
    tc["cls_token"] = {"__type": "AddedToken", "content": "[CLS]", "lstrip": False, "normalized": True, "rstrip": False,
                       "single_word": False}
    tc["sep_token"] = {"content": "[SEP]"}
    del tc["unk_token"]
    spec = read_snapshot_spec(_write(tmp_path, files))
    assert (spec["cls_token"], spec["sep_token"], spec["unk_token"]) == ("[CLS]", "[SEP]", "[UNK]")


def test_no_sentence_bert_config_caps_at_positions_minus_two(tmp_path):
    files = mpnet_layout()
    files["sentence_bert_config.json"] = None
    del files["tokenizer_config.json"]["model_max_length"]
    assert read_snapshot_spec(_write(tmp_path, files))["max_length"] == 512


def test_bert_spec_is_unchanged(tmp_path):
    """a BERT snapshot's spec has no MPNet keys"""
    assert set(read_snapshot_spec(_write(tmp_path, sn.layout("minilm"), vocab=sn.VOCAB))) == \
        {"pooling", "max_length", "do_lower_case", "query_instruction"}


REFUSALS = [
    ("buckets 16", dict(config=dict(MPNET_BASE, relative_attention_num_buckets=16)), "config.json"),
    ("buckets absent", dict(config={k: v for k, v in MPNET_BASE.items() if k != "relative_attention_num_buckets"}), "config.json"),
    ("gelu_new", dict(config=dict(MPNET_BASE, hidden_act="gelu_new")), "config.json"),
    ("head dim 48", dict(config=dict(MPNET_BASE, num_attention_heads=16)), "config.json"),
    ("513 tokens at 514 positions", dict(sbc={"max_seq_length": 513, "do_lower_case": False}), "sentence_bert_config.json"),
    ("cls special not in vocab", dict(vocab=[t for t in VOCAB if t != "<s>"]), "vocab.txt"),
    ("sep special not in vocab", dict(tc_edit={"sep_token": {"content": "<sep>"}}), "vocab.txt"),
    ("unk special not in vocab", dict(tc_edit={"unk_token": "<oov>"}), "vocab.txt"),
]


@pytest.mark.parametrize("label,edit,file", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_mpnet_refusals_name_their_file(tmp_path, label, edit, file):
    files = mpnet_layout(config=edit.get("config"))
    if "sbc" in edit:
        files["sentence_bert_config.json"] = edit["sbc"]
    files["tokenizer_config.json"].update(edit.get("tc_edit", {}))
    with pytest.raises(ValueError) as e:
        read_snapshot_spec(_write(tmp_path, files, vocab=edit.get("vocab", VOCAB)))
    assert os.path.join(str(tmp_path / "snap"), file) in str(e.value), str(e.value)


def test_bucket_refusal_comes_first(tmp_path):
    """the bucket count is checked before any other file of the snapshot is read (here modules.json is refused too)"""
    files = mpnet_layout(config=dict(MPNET_BASE, relative_attention_num_buckets=64))
    files["modules.json"] = files["modules.json"][:1]
    with pytest.raises(ValueError, match=r"config\.json: model_type 'mpnet'"):
        read_snapshot_spec(_write(tmp_path, files))


# ------------------------------------------------------------------------------------------------ tensor names
SMALL = dict(MPNET_BASE, num_hidden_layers=2, hidden_size=128, num_attention_heads=4, intermediate_size=256, vocab_size=len(VOCAB))


@pytest.mark.parametrize("prefix", ["", "mpnet."])
def test_mpnet_state_maps_onto_k5_names(tmp_path, prefix):
    """every tensor of a transformers MPNetModel except pooler.* lands on a name K5 loads, and every name K5 needs but the
    token-type table (which from_pretrained supplies) is there"""
    pytest.importorskip("transformers")
    import bench
    from transformers import MPNetConfig, MPNetModel
    m = MPNetModel(MPNetConfig(**SMALL))
    state = {prefix + k: v.detach().float().numpy() for k, v in m.state_dict().items()}
    d = sn.write(tmp_path / "w", {}, vocab=None, state=state)
    got = E.load_state(d)
    want = set(bench.random_bert_state(SMALL)) - {"embeddings.token_type_embeddings.weight"} | {E.MPNET_REL_BIAS}
    assert {k for k in got if not k.startswith("pooler.") and not k.endswith("position_ids")} == want
    assert got[E.MPNET_REL_BIAS].shape == (32, SMALL["num_attention_heads"])
    np.testing.assert_array_equal(got["encoder.layer.1.attention.self.value.weight"], state[prefix + "encoder.layer.1.attention.attn.v.weight"])
    np.testing.assert_array_equal(got["encoder.layer.0.attention.output.LayerNorm.bias"], state[prefix + "encoder.layer.0.attention.LayerNorm.bias"])


def test_from_pretrained_refuses_an_mpnet_state_without_the_bias(tmp_path):
    """an MPNet snapshot whose weights lack encoder.relative_attention_bias.weight is refused naming it, before any GPU work"""
    import bench
    state = bench.random_bert_state(dict(SMALL, max_position_embeddings=514))
    d = sn.write(tmp_path / "s", mpnet_layout(config=SMALL), vocab=VOCAB, state=state)
    with pytest.raises(ValueError, match="encoder.relative_attention_bias.weight"):
        E.GpuBertEmbedding.from_pretrained(None, d)


# ------------------------------------------------------------------------------------------------ tokenizer
LITERALS = ("<s>", "</s>", "<pad>", "<unk>", "<mask>", "[unk]", "[cls]", "[sep]", "[pad]", "[mask]")


def _fuzz_texts():
    """the fuzz texts of tests/test_wordpiece.py and tests/test_text_native.py, without literal special strings"""
    import random
    from tests.test_text_native import _texts
    from tests.test_wordpiece import TEXTS as WP_TEXTS
    rnd = random.Random(1234)
    alphabet = list("abcdefghijklmnopqrstuvwxyz") + list("ABCXYZ") + list("0123456789") + list(" \t\n  ") + \
        list(".,!?'-()[]$%&/;:@_~<>") + list("éèüñçÅøß") + list("中文日本語") + ["​", "­", "\x00", "\x07", "�", "é", "　", "İ", "ǅ"]
    texts = ["".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 60))) for _ in range(400)]
    texts += ["a" * 101, "a" * 100, "ab" * 60 + " cd", " ".join(["ing"] * 700), "x" * 99 + "é", "the quick fox " * 200]
    texts += _texts(5, 400, 30) + list(WP_TEXTS)
    return [t for t in texts if not any(s in t.lower() for s in LITERALS)]


def _vocab():
    from tests.test_text_native import _vocab as tn_vocab
    toks = ["<s>", "<pad>", "</s>", "<unk>"] + tn_vocab(3)
    toks += [t for t in ("é", "##é", "ü", "中", "文", "日", "本", "語", "ing", "##ion", "the", "quick", "fox") if t not in toks]
    return toks + ["<mask>"]


@pytest.mark.parametrize("lower", [True, False])
def test_wordpiece_with_mpnet_specials_matches_mpnet_tokenizer(tmp_path, lower):
    transformers = pytest.importorskip("transformers")
    p = tmp_path / "vocab.txt"
    vocab = _vocab()
    p.write_text("\n".join(vocab) + "\n", encoding="utf-8")
    ref = transformers.MPNetTokenizer(vocab=str(p), do_lower_case=lower)
    mine = WordPieceTokenizer.from_file(str(p), do_lower_case=lower, max_length=384, **SPECIALS)
    assert mine._nat is not None
    texts = _fuzz_texts()
    want = [ref.encode(t, add_special_tokens=True, truncation=True, max_length=384) for t in texts]
    assert any(len(w) == 384 for w in want) and any(vocab.index("[UNK]") in w for w in want)
    assert all(w[0] == vocab.index("<s>") and w[-1] == vocab.index("</s>") for w in want)
    for t, w in zip(texts, want):
        assert mine.encode_py(t) == w, repr(t)
    assert mine.encode_batch(texts) == want                     # ASCII texts: the native encoder
    flat, offs = mine.encode_batch_flat([t for t in texts if t.isascii()])
    assert [flat[offs[i]:offs[i + 1]].tolist() for i in range(len(offs) - 1)] == [w for t, w in zip(texts, want) if t.isascii()]


def test_literal_specials_are_text(tmp_path):
    """"<s>" typed in a text is WordPiece text here ('<', 's', '>'); transformers' MPNetTokenizer matches it as the added
    token <s> instead (DESIGN.md section 6)"""
    transformers = pytest.importorskip("transformers")
    p = tmp_path / "vocab.txt"
    p.write_text("\n".join(VOCAB + ["<", ">", "s", "/"]) + "\n", encoding="utf-8")
    mine = WordPieceTokenizer.from_file(str(p), **SPECIALS)
    ids = {t: i for i, t in enumerate(VOCAB + ["<", ">", "s", "/"])}
    assert mine.encode("the <s> fox") == mine.encode_py("the <s> fox") == \
        [ids["<s>"], ids["the"], ids["<"], ids["s"], ids[">"], ids["fox"], ids["</s>"]]
    ref = transformers.MPNetTokenizer(vocab=str(p))
    assert ref.encode("the <s> fox") == [ids["<s>"], ids["the"], ids["<s>"], ids["fox"], ids["</s>"]]


def test_default_specials_keep_the_bert_ids(tmp_path):
    p = tmp_path / "vocab.txt"
    p.write_text("\n".join(sn.VOCAB) + "\n", encoding="utf-8")
    a = WordPieceTokenizer.from_file(str(p))
    b = WordPieceTokenizer.from_file(str(p), cls_token="[CLS]", sep_token="[SEP]", unk_token="[UNK]")
    t = "The quick brown fox jumps over zzz"
    assert a.encode(t) == b.encode(t) == a.encode_py(t) and a.encode(t)[0] == sn.VOCAB.index("[CLS]")
