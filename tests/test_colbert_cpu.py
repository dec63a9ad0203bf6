"""ColBERT snapshot reading and tokenisation without a GPU: read_colbert_spec on synthetic Stanford and PyLate snapshots
(and each field it refuses), and the query / passage ids and skiplist against a plain restatement on transformers'
BertTokenizer (". " + text, position 1 overwritten by the marker, truncation, [MASK] padding)."""
import json
import os
import string

import numpy as np
import pytest

from tests import st_snapshot as sts

VOCAB = sts.VOCAB + ["[unused0]", "[unused1]", ";", "(", ")", "#"]
BERT = dict(sts.BGE_SMALL, vocab_size=len(VOCAB), architectures=["HF_ColBERT"])
META = {"query_maxlen": 32, "doc_maxlen": 12, "dim": 96, "mask_punctuation": True, "attend_to_mask_tokens": False,
        "query_token_id": "[unused0]", "doc_token_id": "[unused1]", "similarity": "cosine"}


def _stanford(path, **meta):
    sts.write(path, {"config.json": BERT, "tokenizer_config.json": {"do_lower_case": True}}, vocab=VOCAB)
    with open(os.path.join(path, "artifact.metadata"), "w") as f:
        json.dump(dict(META, **meta), f)
    return str(path)


def _pylate(path, dense=None, st=None):
    sts.write(path, {"config.json": dict(BERT, architectures=["BertModel"]), "tokenizer_config.json": {"do_lower_case": True},
                     "modules.json": [{"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
                                      {"idx": 1, "name": "1", "path": "1_Dense", "type": "pylate.models.Dense.Dense"}],
                     "1_Dense/config.json": dict({"in_features": 384, "out_features": 128, "bias": False,
                                                  "activation_function": "torch.nn.modules.linear.Identity"}, **(dense or {})),
                     "config_sentence_transformers.json": dict({"query_prefix": "[unused0]", "document_prefix": "[unused1]",
                                                                "query_length": 32, "document_length": 180,
                                                                "attend_to_expansion_tokens": False, "do_query_expansion": True,
                                                                "skiplist_words": list(string.punctuation)}, **(st or {}))},
              vocab=VOCAB)
    return str(path)


def test_reads_stanford_and_pylate(tmp_path):
    from kaito_b200.rerank import is_colbert_snapshot, read_colbert_spec
    s = read_colbert_spec(_stanford(tmp_path / "s"))
    assert (s["query_maxlen"], s["doc_maxlen"], s["dim"], s["attend_to_mask_tokens"], s["mask_punctuation"]) == (32, 12, 96, False, True)
    assert (s["q_marker"], s["d_marker"]) == (VOCAB.index("[unused0]"), VOCAB.index("[unused1]"))
    p = read_colbert_spec(_pylate(tmp_path / "p"))
    assert (p["query_maxlen"], p["doc_maxlen"], p["dim"]) == (32, 180, 128) and p["weight"][0].endswith(os.path.join("1_Dense", "pytorch_model.bin"))
    assert is_colbert_snapshot(str(tmp_path / "s")) and is_colbert_snapshot(str(tmp_path / "p"))
    sts.write(tmp_path / "ce", sts.layout("bge"))
    assert not is_colbert_snapshot(str(tmp_path / "ce"))


@pytest.mark.parametrize("meta, field", [({"similarity": "l2"}, "similarity"), ({"query_token_id": "[Q]"}, "query_token_id"),
                                         ({"doc_token_id": "[nope]"}, "doc_token_id"), ({"query_maxlen": 64}, "query_maxlen"),
                                         ({"dim": 100}, "dim"), ({"attend_to_mask_tokens": "no"}, "attend_to_mask_tokens"),
                                         ({"interaction": "flipr"}, "interaction")])
def test_refuses_stanford_fields(tmp_path, meta, field):
    from kaito_b200.rerank import read_colbert_spec
    with pytest.raises(ValueError, match=f"artifact.metadata: {field}"):
        read_colbert_spec(_stanford(tmp_path, **meta))


@pytest.mark.parametrize("dense, st, where", [({"bias": True}, None, "config.json: bias"),
                                              ({"activation_function": "torch.nn.modules.activation.Tanh"}, None, "activation_function"),
                                              ({"in_features": 768}, None, "in_features"),
                                              (None, {"do_query_expansion": False}, "do_query_expansion"),
                                              (None, {"query_prefix": "[Q] "}, "query_prefix")])
def test_refuses_pylate_fields(tmp_path, dense, st, where):
    from kaito_b200.rerank import read_colbert_spec
    with pytest.raises(ValueError, match=where.replace("[", r"\[")):
        read_colbert_spec(_pylate(tmp_path, dense, st))


def test_refuses_pylate_module_order(tmp_path):
    from kaito_b200.rerank import read_colbert_spec
    path = _pylate(tmp_path)
    with open(os.path.join(path, "modules.json"), "w") as f:
        json.dump([{"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Pooling"},
                   {"idx": 1, "name": "1", "path": "1_Dense", "type": "pylate.models.Dense.Dense"}], f)
    with pytest.raises(ValueError, match="modules.json"):
        read_colbert_spec(path)


def test_refuses_a_projection_bias_in_the_dense_weights(tmp_path):
    """PyLate keeps the projection in the Dense module's own file: a bias there is refused, naming that file"""
    import numpy as np
    from safetensors.numpy import save_file
    from kaito_b200.rerank import GpuLateInteractionReranker
    path = _pylate(tmp_path)
    save_file({"linear.weight": np.zeros((128, 384), np.float32), "linear.bias": np.zeros(128, np.float32)},
              os.path.join(path, "1_Dense", "model.safetensors"))
    save_file({"embeddings.word_embeddings.weight": np.zeros((len(VOCAB), 384), np.float32)}, os.path.join(path, "model.safetensors"))
    with pytest.raises(ValueError, match=r"1_Dense.model\.safetensors: tensor linear\.bias"):
        GpuLateInteractionReranker.from_pretrained(None, path)


def test_refuses_non_bert_config(tmp_path):
    from kaito_b200.rerank import read_colbert_spec
    path = _stanford(tmp_path)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(dict(BERT, hidden_act="relu"), f)
    with pytest.raises(ValueError, match="config.json: hidden_act"):
        read_colbert_spec(path)


TEXTS = ["", "the quick brown fox", "The quick, brown fox! jump's over the lazy dog?", " ".join(["quick brown fox"] * 20),
         "!!! ... ?", "token ; ( gpu ) # search"]


@pytest.mark.parametrize("attend", [False, True])
def test_ids_match_bert_tokenizer(tmp_path, attend):
    from transformers import BertTokenizer
    from kaito_b200.rerank import colbert_query_ids, colbert_skip_ids
    from kaito_b200.text import WordPieceTokenizer
    path = _stanford(tmp_path)
    hf = BertTokenizer(os.path.join(path, "vocab.txt"), do_lower_case=True)
    tok = WordPieceTokenizer(VOCAB)
    q_marker, d_marker, mask = VOCAB.index("[unused0]"), VOCAB.index("[unused1]"), VOCAB.index("[MASK]")
    ids, keys = colbert_query_ids(tok, TEXTS, 32, q_marker, mask, attend)
    for t, got, k in zip(TEXTS, ids, keys):
        enc = hf([". " + t], padding="max_length", truncation=True, max_length=32)
        want = np.asarray(enc["input_ids"][0]); att = np.asarray(enc["attention_mask"][0])
        want[1] = q_marker
        want[want == hf.pad_token_id] = mask
        assert got.tolist() == want.tolist(), t
        assert k == (32 if attend else int(att.sum()))
    # the skiplist: the first id of each string.punctuation character, as ColBERT builds it
    want_skip = sorted({hf.encode(c, add_special_tokens=False)[0] for c in string.punctuation})
    assert colbert_skip_ids(tok, None).tolist() == want_skip


def test_passage_ids_and_keep_mask(tmp_path):
    from transformers import BertTokenizer
    from kaito_b200.rerank import GpuLateInteractionReranker, colbert_skip_ids
    from kaito_b200.text import WordPieceTokenizer
    path = _stanford(tmp_path)
    hf = BertTokenizer(os.path.join(path, "vocab.txt"), do_lower_case=True)
    r = GpuLateInteractionReranker.__new__(GpuLateInteractionReranker)       # the host side alone: no engine
    r.tokenizer = WordPieceTokenizer(VOCAB)
    r.spec = {"doc_maxlen": 12, "d_marker": VOCAB.index("[unused1]")}
    r.skip = colbert_skip_ids(r.tokenizer, None)
    skip = {hf.encode(c, add_special_tokens=False)[0] for c in string.punctuation}
    for t, (ids, keep) in zip(TEXTS, r.encode_passages(TEXTS)):
        want = hf([". " + t], truncation=True, max_length=12)["input_ids"][0]
        want[1] = VOCAB.index("[unused1]")
        assert ids.tolist() == want, t
        assert keep.tolist() == [0 if x in skip else 1 for x in want], t
    all_punct = r.encode_passages(["!!! ... ?"])[0]
    assert all_punct[1].tolist() == [1, 1, 0, 0, 0, 0, 0, 0, 0, 1]          # [CLS] [D] and [SEP] stay


# ------------------------------------------------------------------------------------ the fmaf yardstick
def _round_f32(x):
    """the Fraction x rounded to the nearest fp32, ties to even (subnormals included), as a Python float"""
    from fractions import Fraction
    if x == 0:
        return 0.0
    sign, x = (-1.0 if x < 0 else 1.0), abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    while Fraction(2) ** e > x:
        e -= 1
    while Fraction(2) ** (e + 1) <= x:
        e += 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    m = x / ulp
    n = m.numerator // m.denominator
    r = m - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2):
        n += 1
    v = n * ulp
    return sign * (float("inf") if v >= 2 ** 128 else float(v))


def _exact_fmaf(a, b, c):
    from fractions import Fraction
    return np.float32(_round_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))))


def _check_fmaf(a, b, c):
    from tests import colbert_reference as cr
    got = cr.fmaf(a, b, c)
    want = np.array([_exact_fmaf(x, y, z) for x, y, z in zip(a, b, c)], np.float32)
    bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
    assert not len(bad), [(float(a[i]), float(b[i]), float(c[i]), float(got[i]), float(want[i])) for i in bad[:5]]


@pytest.mark.skipif(np.finfo(np.longdouble).nmant < 63, reason="needs a 64-bit long double significand")
def test_fmaf_emulation_is_one_rounding_on_random_triples():
    """tests/colbert_reference.fmaf (the yardstick of the exact MaxSim tests) against a Fraction fma rounded once to fp32:
    unit-vector components (the kernel's operands) and accumulators of all sizes, and triples whose product is far above
    or far below the addend, so the exact sum needs more than 64 bits"""
    g = np.random.default_rng(0)
    n = 6000
    a = (g.standard_normal(n) / 8).astype(np.float32)
    b = (g.standard_normal(n) / 8).astype(np.float32)
    c = (g.standard_normal(n) * np.exp2(g.integers(-40, 12, n))).astype(np.float32)
    _check_fmaf(a, b, c)
    e = np.exp2(g.integers(-60, 60, (3, n)))
    _check_fmaf(*[(g.standard_normal(n) * e[i]).astype(np.float32) for i in range(3)])


@pytest.mark.skipif(np.finfo(np.longdouble).nmant < 63, reason="needs a 64-bit long double significand")
def test_fmaf_emulation_near_fp32_midpoints():
    """addends c of both parities and signs, and products that put c + a b exactly on the midpoint to c's neighbour (ties
    to even), or 2^-k of an ulp to either side of it for k = 2 .. 24; fmaf(a, b, -fl(a b)) (the product's exact rounding
    error); and the limit of the yardstick: a sum 2^-47 ulp below a midpoint, which the 64-bit intermediate rounds onto
    the midpoint, so the emulation rounds an odd c the wrong way -- the error class of about 2^-40 the exact tests accept"""
    g = np.random.default_rng(1)
    cs = (g.standard_normal(64) * np.exp2(g.integers(-20, 20, 64))).astype(np.float32)
    bits = cs.view(np.int32)
    bits[::2] |= 1                                                 # odd significands ...
    bits[1::2] &= ~1                                               # ... and even ones
    assert (bits[::2] % 2 == 1).all() and (bits[1::2] % 2 == 0).all()
    cs = np.concatenate([cs, -cs])
    a, b, c = [], [], []
    for x in cs:
        half = np.float32(np.spacing(np.abs(x)) / 2) * np.sign(x)    # towards the neighbour away from zero
        for k in range(2, 25):
            for f in (1.0, 1.0 + 2.0 ** -(k - 1), 1.0 - 2.0 ** -(k - 1)):
                a.append(half); b.append(np.float32(f)); c.append(x)
        a.append(half); b.append(np.float32(-1.0)); c.append(x)     # the midpoint towards zero
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    assert np.isfinite(a * b).all()
    _check_fmaf(a, b, c)
    p, q = (g.standard_normal((2, 2000)) / 8).astype(np.float32)
    _check_fmaf(p, q, -(p * q))
    from tests import colbert_reference as cr
    for x in (np.float32(1.0), np.float32(1.0 + 2.0 ** -23)):
        u = np.float32(np.spacing(x))
        a1, b1 = np.float32(u / 2 * np.float32(1 + 2.0 ** -23)), np.float32(1 - 2.0 ** -23)   # a b = u / 2 (1 - 2^-46)
        want, got = _exact_fmaf(a1, b1, x), cr.fmaf(a1, b1, x)
        assert want == x
        assert got == (x if x.view(np.int32) % 2 == 0 else np.nextafter(x, np.float32(2)))
