"""GPU tests of XLM-RoBERTa cross-encoders (bge-reranker-base / -large / -v2-m3 shapes) through krag_rerank: positions
from pad_token_id + 1 (krag_embedder_set_position_offset), unsegmented pairs <s> q </s></s> d </s> (seg_b = NULL), and the
classifier.dense / out_proj head loaded as BERT's pooler and classifier.

Logits are held to an fp64 transformers.XLMRobertaForSequenceClassification run on each pair alone, by the rules of the
BERT cross-encoder tests: the default mode within F = 40 times torch fp32's own error and 1e-4 on the sigmoid score
(test_gpu_rerank.py), the fp16 mode within torch bf16 autocast's error (test_gpu_rerank_fp16.py) and SCORE_TOL_FP16_XLMR on
the sigmoid score.  Random and stressed weights (no checkpoints offline); KRAG_TEST_BGE_RERANKER_DIR points the last test at
a real snapshot."""
import os

import numpy as np
import pytest

from tests import bert_reference as br
from tests import xlmr_reference as xr
from tests.test_gpu_rerank import F, SCORE_TOL

CLS, SEP = 0, 2
# fp16 mode, sigmoid score: about twice the worst error measured here, 1.8e-3 at bge-reranker-large full depth and 1.7e-3 at
# -base (random weights; logit errors 0.06-0.36x torch bf16 autocast's).  The 1.2e-3 of test_gpu_rerank_fp16.py was measured
# at BERT cross-encoder shapes of at most 12 x 384; 12 and 24 layers of 768 and 1024 accumulate more fp16 operand rounding.
SCORE_TOL_FP16_XLMR = 4e-3
# (label, shape, layers (None: full depth), regimes, queries x passages, passage length range, long pair length)
CASES = [
    ("base", "bge-reranker-base", None, ("random", "stressed"), (4, 8), (0, 200), 512),
    ("large short", "bge-reranker-large", None, ("random",), (3, 6), (0, 60), 0),
    ("large 512", "bge-reranker-large", 4, ("random", "stressed"), (3, 6), (0, 200), 512),
    ("v2-m3 8k", "bge-reranker-v2-m3", 2, ("random",), (2, 3), (0, 100), 8190),
]


def _cfg(shape, layers):
    cfg = xr.encoder_config(shape)
    if layers:
        cfg["num_hidden_layers"] = layers
    return cfg


def _encoder(ctx, cfg, state, precision="fp32"):
    from kaito_b200 import _native
    e = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                         cfg["vocab_size"], cfg["max_position_embeddings"], 1, 1e-5)
    e.load_state_dict(state, head=True)
    e.set_position_offset(xr.PAD + 1)
    e.set_precision(precision)
    return e


def _ids(g, n, vocab):
    """n content ids, never the pad id (transformers numbers a pad token's position differently), the top id included"""
    t = g.integers(4, vocab, n).astype(np.int32)
    if n > 2:
        t[n // 2] = vocab - 1
    return t


def _pairs(g, cfg, nq, per_q, d_len, long_len):
    """packed unsegmented pairs (flat, toff, poff): per query, passages of d_len tokens, the first one long_len tokens in
    all (when set), an empty query and an empty passage at the end"""
    from kaito_b200.rerank import build_pairs
    V = cfg["vocab_size"]
    max_length = max(long_len, 512)
    qs, ds = [], []
    for i in range(nq):
        q = _ids(g, int(g.integers(1, 24)), V)
        qs.append((q, len(q)))
        cands = []
        for j in range(per_q):
            n = long_len - 4 - len(q) if long_len and j == 0 and i == 0 else int(g.integers(*d_len))
            d = _ids(g, n, V)
            cands.append((d, n))
        ds.append(cands)
    qs.append((np.zeros(0, np.int32), 0))
    ds.append([(np.zeros(0, np.int32), 0), (_ids(g, 7, V), 7)])
    flat, toff, seg, poff = build_pairs(CLS, SEP, qs, ds, max_length, 2)
    assert seg is None and (not long_len or int(np.diff(toff).max()) == long_len)
    return flat, toff, poff


def _all_scores(enc, flat, toff, poff, act):
    n_max = int(np.diff(poff).max())
    pos, sc = enc.rerank(poff, flat, toff, None, n_max, act)
    out = np.empty(int(poff[-1]), np.float32)
    for q in range(len(poff) - 1):
        n = int(poff[q + 1] - poff[q])
        assert sorted(pos[q, :n].tolist()) == list(range(n)) and (pos[q, n:] == -1).all()
        out[poff[q] + pos[q, :n]] = sc[q, :n]
    return out, pos


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


@pytest.mark.gpu
@pytest.mark.parametrize("label,shape,layers,regimes,qp,d_len,long_len", CASES, ids=[c[0] for c in CASES])
def test_logits_match_fp64(ctx, label, shape, layers, regimes, qp, d_len, long_len):
    from kaito_b200 import _native
    cfg = _cfg(shape, layers)
    for regime in regimes:
        state = xr.k5_state(cfg, regime, seed=len(label))
        ref = xr.Fp64XlmrCrossEncoder(cfg, state, device="cuda")
        flat, toff, poff = _pairs(np.random.default_rng(len(label) + 1), cfg, *qp, d_len, long_len)
        n = len(toff) - 1
        lens = np.diff(toff)
        idx = sorted(set(br.sample(lens.tolist(), 10).tolist()) | {n - 1, n - 2, int(lens.argmax())})
        pairs = [flat[toff[i]:toff[i + 1]] for i in idx]
        ref.range_max = 0.0
        l64, l32 = ref.logits(pairs)
        br.check_range(ref.range_max)
        b16 = ref.logits_bf16(pairs)
        for precision in ("fp32", "fp16"):
            enc = _encoder(ctx, cfg, state, precision)
            logit, _ = _all_scores(enc, flat, toff, poff, _native.RERANK_IDENTITY)
            score, pos = _all_scores(enc, flat, toff, poff, _native.RERANK_SIGMOID)
            enc.destroy()
            k5 = float(np.abs(logit[idx] - l64).max())
            ds = float(np.abs(score[idx] - _sigmoid(l64)).max())
            t32, t16 = float(np.abs(l32 - l64).max()), float(np.abs(b16 - l64).max())
            print(f"xlmr rerank {precision} vs fp64 | {label} {regime} | {len(idx)} of {n} pairs, {int(toff[-1])} tok, longest "
                  f"{int(lens.max())} | logit err {k5:.2e} | torch fp32 {t32:.2e} | torch bf16 {t16:.2e} | sigmoid err {ds:.2e} | "
                  f"Linear range {ref.range_max:.3g}")
            if precision == "fp32":
                assert k5 / max(t32, 2.0 ** -23) <= F, (label, regime, k5, t32)
                assert ds <= SCORE_TOL, (label, regime, ds)
                bound = SCORE_TOL
            else:
                assert k5 <= t16, (label, regime, k5, t16)
                assert ds <= SCORE_TOL_FP16_XLMR, (label, regime, ds)
                bound = SCORE_TOL_FP16_XLMR
            # the per-query order of the scored pairs follows fp64 wherever neighbours are further apart than twice the bound
            s64 = {i: s for i, s in zip(idx, _sigmoid(l64))}
            for q in range(len(poff) - 1):
                a, b = int(poff[q]), int(poff[q + 1])
                ranked = [a + int(p) for p in pos[q, :b - a] if a + int(p) in s64]
                for x, y in zip(ranked, ranked[1:]):
                    assert s64[x] >= s64[y] - 2 * bound, (label, regime, precision, q, x, y)


@pytest.mark.gpu
def test_unsegmented_pairs_and_the_position_offset(ctx):
    """seg_b = NULL on a type_vocab = 1 model; with offset 2 a pair of max_position - 2 tokens runs and one of
    max_position - 1 is KRAG_E_INVALID; a captured graph follows a change of the offset"""
    from kaito_b200 import _native
    cfg = dict(num_hidden_layers=2, hidden_size=256, num_attention_heads=4, intermediate_size=1024, vocab_size=1000,
               max_position_embeddings=514, type_vocab_size=1)
    state = xr.k5_state(cfg, "random", seed=3)
    enc = _encoder(ctx, cfg, state)
    g = np.random.default_rng(4)
    ok = np.concatenate([[CLS], _ids(g, 510, 1000), [SEP]]).astype(np.int32)          # 512 = max_position - 2
    pos, sc = enc.rerank(np.array([0, 1], np.int32), ok, np.array([0, 512], np.int32), None, 1, _native.RERANK_IDENTITY)
    ref = xr.Fp64XlmrCrossEncoder(cfg, state, device="cuda")
    l64, l32 = ref.logits([ok])
    assert pos[0, 0] == 0 and abs(float(sc[0, 0]) - l64[0]) <= F * max(abs(l32[0] - l64[0]), 2.0 ** -23)
    long = np.concatenate([ok, [SEP]]).astype(np.int32)
    with pytest.raises(_native.KragError) as e:
        enc.rerank(np.array([0, 1], np.int32), long, np.array([0, 513], np.int32), None, 1)
    assert e.value.code == _native.KRAG_E_INVALID
    with pytest.raises(_native.KragError) as e:                      # token types need a second row
        enc.rerank(np.array([0, 1], np.int32), ok, np.array([0, 512], np.int32), np.array([5], np.int32), 1)
    assert e.value.code == _native.KRAG_E_INVALID
    with pytest.raises(_native.KragError):
        enc.set_position_offset(-1)
    # one shape three times at offset 2 (the second and third replay a captured graph), then at offset 0: the replay must
    # take the new positions, as a fresh embedder at offset 0 computes them
    short = [np.concatenate([[CLS], _ids(g, 30, 1000), [SEP, SEP], _ids(g, 40, 1000), [SEP]]).astype(np.int32) for _ in range(8)]
    flat, toff = np.concatenate(short), np.arange(9, dtype=np.int32) * len(short[0])
    poff = np.array([0, 8], np.int32)
    at2 = [enc.rerank(poff, flat, toff, None, 8, _native.RERANK_IDENTITY)[1] for _ in range(3)]
    enc.set_position_offset(0)
    at0 = [enc.rerank(poff, flat, toff, None, 8, _native.RERANK_IDENTITY)[1] for _ in range(2)]
    fresh = _encoder(ctx, cfg, state)
    fresh.set_position_offset(0)
    want0 = fresh.rerank(poff, flat, toff, None, 8, _native.RERANK_IDENTITY)[1]
    assert np.array_equal(at2[0], at2[1]) and np.array_equal(at2[0], at2[2])
    assert np.array_equal(at0[0], want0) and np.array_equal(at0[1], want0) and not np.array_equal(at0[0], at2[0])
    enc.destroy(); fresh.destroy()


@pytest.mark.gpu
def test_from_pretrained_and_store_retrieve(ctx, tmp_path):
    """a bge-reranker-shaped snapshot (trained tokenizer, random weights) through GpuCrossEncoder.from_pretrained and the
    store's retrieve: the returned ids are the fused candidates reordered by the fp64 scores"""
    from kaito_b200.embedding import HashingEmbedding
    from kaito_b200.rerank import GpuCrossEncoder, build_pairs
    from kaito_b200.vector_store import VectorStore, embed_text
    tok_dir = xr.train_tokenizer(str(tmp_path / "tok"), seed=0)
    conf = xr.config_json("bge-reranker-base", num_hidden_layers=2, vocab_size=1000)
    cfg = _cfg("bge-reranker-base", 2)
    cfg["vocab_size"] = 1000
    state = xr.k5_state(cfg, "random", seed=6)
    snap = xr.write_snapshot(str(tmp_path / "snap"), conf, tok_dir, state=xr.hf_state(state))
    ce = GpuCrossEncoder.from_pretrained(ctx, snap)
    assert ce.activation == "sigmoid" and ce.max_length == 512 and ce.specials == 4
    g = np.random.default_rng(2)
    docs = [{"text": " ".join(g.choice(xr.WORDS, int(g.integers(5, 60)))), "metadata": {"n": str(i % 3)}} for i in range(200)]
    plain = VectorStore(HashingEmbedding(384), ctx)
    rr = VectorStore(HashingEmbedding(384), ctx, reranker=ce)
    plain.index_documents("x_plain", docs); rr.index_documents("x_rr", docs)
    ref = xr.Fp64XlmrCrossEncoder(cfg, state, device="cuda")
    for query in ("quick brown fox", "gpu token retrieval café", "日本語 москва"):
        got = rr.retrieve("x_rr", query, max_node_count=10)
        fused = plain.retrieve("x_plain", query, max_node_count=30)["results"]
        assert got["count"] == 10 and len(fused) == 30
        by_id = {n.node_id: n for n in plain.index_map["x_plain"].nodes}
        texts = [embed_text(r["text"], by_id[r["node_id"]].metadata) for r in fused]
        q = ce.tokenizer.encode_batch_plain([query])[0]
        flat, toff, _, _ = build_pairs(CLS, SEP, [(q, len(q))], [ce.encode_passages(texts)], 512, 2)
        s64 = _sigmoid(ref.logits([flat[toff[i]:toff[i + 1]] for i in range(30)])[0])
        want = np.lexsort((np.arange(30), -s64))[:10]
        ids = [r["node_id"] for r in got["results"]]
        for j, w in enumerate(want):
            if ids[j] != fused[w]["node_id"]:        # only a near-tie may swap
                other = [r["node_id"] for r in fused].index(ids[j])
                assert abs(s64[other] - s64[w]) < 2 * SCORE_TOL, (query, j)
        assert np.allclose([r["score"] for r in got["results"]], np.sort(s64)[::-1][:10], atol=SCORE_TOL)


@pytest.mark.gpu
@pytest.mark.skipif(not os.getenv("KRAG_TEST_BGE_RERANKER_DIR"), reason="set KRAG_TEST_BGE_RERANKER_DIR to a bge-reranker snapshot")
def test_real_bge_reranker_snapshot(ctx):
    """a real checkpoint (its activations' range is only known from one): tokenizer ids against the Rust tokenizer, logits
    against transformers in fp64, and every Linear operand inside the fp16 range"""
    import torch
    from tokenizers import Tokenizer
    from transformers import XLMRobertaForSequenceClassification
    from kaito_b200 import _native
    from kaito_b200.rerank import GpuCrossEncoder, build_pairs
    snap = os.environ["KRAG_TEST_BGE_RERANKER_DIR"]
    ce = GpuCrossEncoder.from_pretrained(ctx, snap)
    rust = Tokenizer.from_file(os.path.join(snap, "tokenizer.json"))
    queries = ["what is panda?", "Wie hoch ist der Eiffelturm?", "北京的人口是多少", ""]
    passages = ["The giant panda is a bear species endemic to China.", "Der Eiffelturm ist 330 Meter hoch.",
                "北京市常住人口约2189万人。", "hi", "", "Paris is the capital of France. " * 60]
    for t in queries + passages:
        assert ce.tokenizer.encode_batch_plain([t])[0].tolist() == rust.encode(t, add_special_tokens=False).ids, t
    qs = [(q, len(q)) for q in ce.tokenizer.encode_batch_plain(queries)]
    ds = [ce.encode_passages(passages)] * len(queries)
    flat, toff, _, poff = build_pairs(CLS, SEP, qs, ds, ce.max_length, 2)
    m = XLMRobertaForSequenceClassification.from_pretrained(snap, attn_implementation="eager").double().eval().cuda()
    rng = [0.0]
    for mod in m.modules():
        if isinstance(mod, torch.nn.Linear):
            mod.register_forward_hook(lambda mod, i, o: rng.__setitem__(0, max(rng[0], float(i[0].abs().max()), float(o.abs().max()))))
    with torch.no_grad():
        l64 = np.array([float(m(input_ids=torch.tensor(flat[toff[i]:toff[i + 1]][None].astype(np.int64)).cuda()).logits[0, 0])
                        for i in range(len(toff) - 1)])
    br.check_range(rng[0])
    ce._emb.set_precision("fp32")
    got, _ = _all_scores(ce._emb, flat, toff, poff, _native.RERANK_SIGMOID)
    print(f"real bge-reranker: sigmoid err {float(np.abs(got - _sigmoid(l64)).max()):.2e}, Linear range {rng[0]:.3g}")
    assert float(np.abs(got - _sigmoid(l64)).max()) <= SCORE_TOL
