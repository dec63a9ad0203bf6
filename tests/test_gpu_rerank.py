"""GPU tests of cross-encoder reranking (krag_rerank: K5 with token types, pooler and classifier head, per-query top-k).
Logits are held to an fp64 transformers.BertForSequenceClassification run on each pair alone, by the rule of
test_gpu_embed.py: the error is at most F = 40 times torch fp32's own error against fp64, and the sigmoid score moves by at
most 1e-4.  Random weights (no checkpoints offline): bert_reference's generators plus a pooler and a one-label classifier."""
import numpy as np
import pytest

from tests import bert_reference as br

F = 40.0
SCORE_TOL = 1e-4
CE_MODELS = {   # BertConfig of the cross-encoder checkpoints
    "MiniLM-L6": dict(num_hidden_layers=6, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=30522,
                      max_position_embeddings=512),
    "MiniLM-L12": dict(num_hidden_layers=12, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=30522,
                       max_position_embeddings=512),
    "TinyBERT-L2": dict(num_hidden_layers=2, hidden_size=128, num_attention_heads=2, intermediate_size=512, vocab_size=30522,
                        max_position_embeddings=512),
    "base": dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=30522,
                 max_position_embeddings=512),
}


def _state(cfg, regime, seed=0):
    import bench
    st = br.stressed_state(cfg, seed)[0] if regime == "stressed" else bench.random_bert_state(cfg, seed)
    return br.head_state(cfg, st, seed)


def _encoder(ctx, cfg, state):
    from kaito_b200 import _native
    e = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                         cfg["vocab_size"], cfg["max_position_embeddings"])
    e.load_state_dict(state, head=True)
    return e


def _random_pairs(g, n_queries, per_query, q_len=(0, 30), d_len=(0, 200), long_every=0, max_length=512):
    from kaito_b200.rerank import build_pairs
    qs, ds = [], []
    for i in range(n_queries):
        q = g.integers(1000, 30000, int(g.integers(*q_len) if q_len[1] > q_len[0] else q_len[0])).astype(np.int32)
        qs.append((q, len(q)))
        cands = []
        for j in range(per_query):
            n = 600 if long_every and (i * per_query + j) % long_every == 0 else int(g.integers(*d_len))
            d = g.integers(1000, 30000, n).astype(np.int32)
            cands.append((d[:max_length - 3], n))
        ds.append(cands)
    return build_pairs(2, 3, qs, ds, max_length)


def _all_scores(enc, flat, toff, seg, poff, act):
    """every pair's score (top_k = each query's whole list, put back in pair order)"""
    n_max = int(np.diff(poff).max())
    pos, sc = enc.rerank(poff, flat, toff, seg, n_max, act)
    out = np.empty(int(poff[-1]), np.float32)
    for q in range(len(poff) - 1):
        n = int(poff[q + 1] - poff[q])
        assert sorted(pos[q, :n].tolist()) == list(range(n)) and (pos[q, n:] == -1).all()
        out[poff[q] + pos[q, :n]] = sc[q, :n]
    return out


def _pairs_of(flat, toff, seg, idx):
    return [(flat[toff[i]:toff[i + 1]], int(seg[i])) for i in idx]


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["bench", "stressed"])
@pytest.mark.parametrize("model", list(CE_MODELS))
def test_logits_match_fp64(ctx, model, regime):
    from kaito_b200 import _native
    if model == "base" and regime == "stressed":
        pytest.skip("the stressed regime runs at the MiniLM and TinyBERT shapes")
    cfg = CE_MODELS[model]
    state = _state(cfg, regime)
    enc = _encoder(ctx, cfg, state)
    g = np.random.default_rng(5)
    # 8 queries x 30 pairs, every 37th pair a 512-token one; plus the seg_b edges: an empty query and an empty passage
    flat, toff, seg, poff = _random_pairs(g, 8, 30, long_every=37)
    edge = _random_pairs(g, 2, 3, q_len=(0, 0), d_len=(0, 1))      # empty query, empty passages
    flat = np.concatenate([flat, edge[0]]); toff = np.concatenate([toff, toff[-1] + edge[1][1:]])
    seg = np.concatenate([seg, edge[2]]); poff = np.concatenate([poff, poff[-1] + edge[3][1:]])
    logit = _all_scores(enc, flat, toff, seg, poff, _native.RERANK_IDENTITY)
    score = _all_scores(enc, flat, toff, seg, poff, _native.RERANK_SIGMOID)
    lens = np.diff(toff)
    n = len(lens)
    idx = sorted(set(br.sample(lens.tolist(), 12 if model == "base" else 20).tolist()) | {n - 1, n - 2, n - 6}
                 | set(np.flatnonzero(lens == 512)[:2].tolist()))
    ref = br.Fp64CrossEncoder(cfg, state)
    l64, l32 = ref.logits(_pairs_of(flat, toff, seg, idx))
    got = logit[idx].astype(np.float64)
    k5, t32 = float(np.abs(got - l64).max()), float(np.abs(l32 - l64).max())
    ratio = k5 / max(t32, 2.0 ** -23)
    ds = float(np.abs(score[idx] - 1.0 / (1.0 + np.exp(-l64))).max())
    print(f"rerank vs fp64 | {model} {regime} | {len(idx)} of {n} pairs, {int(toff[-1])} tok | logit err {k5:.2e} | "
          f"torch fp32 {t32:.2e} | ratio {ratio:.2f} | sigmoid err {ds:.2e}")
    assert ratio <= F, (k5, t32, ratio)
    assert ds <= SCORE_TOL, ds
    assert np.array_equal(score, (1.0 / (1.0 + np.exp(-logit.astype(np.float64)))).astype(np.float32)) or \
        float(np.abs(score - 1.0 / (1.0 + np.exp(-logit.astype(np.float64)))).max()) < 1e-6
    enc.destroy()


@pytest.mark.gpu
def test_chunked_call_agrees_with_per_query_calls(ctx):
    from kaito_b200 import _native
    cfg = CE_MODELS["MiniLM-L6"]
    enc = _encoder(ctx, cfg, _state(cfg, "bench"))
    g = np.random.default_rng(9)
    flat, toff, seg, poff = _random_pairs(g, 64, 30, q_len=(4, 20), d_len=(20, 80))
    assert toff[-1] > 65536                                        # more than one forward
    pos, sc = enc.rerank(poff, flat, toff, seg, 10)
    for q in range(0, 64, 7):
        a, b = int(poff[q]), int(poff[q + 1])
        sub_toff = toff[a:b + 1] - toff[a]
        p1, s1 = enc.rerank(np.array([0, b - a], np.int32), flat[toff[a]:toff[b]], sub_toff, seg[a:b], 10)
        assert float(np.abs(s1[0] - sc[q]).max()) <= SCORE_TOL
        gaps = np.diff(-sc[q].astype(np.float64))
        for j in range(10):                 # same ranking where neighbouring scores are further apart than the bound
            if (j == 0 or gaps[j - 1] > 2 * SCORE_TOL) and (j == 9 or gaps[j] > 2 * SCORE_TOL):
                assert p1[0, j] == pos[q, j], (q, j)
    enc.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("n,top_k", [(30, 1), (30, 30), (300, 10), (300, 300)])
def test_selection_order_and_ties(ctx, n, top_k):
    from kaito_b200 import _native
    from kaito_b200.rerank import build_pairs
    cfg = CE_MODELS["TinyBERT-L2"]
    enc = _encoder(ctx, cfg, _state(cfg, "bench"))
    g = np.random.default_rng(n + top_k)
    q = g.integers(1000, 30000, 8).astype(np.int32)
    uniq = [g.integers(1000, 30000, int(g.integers(1, 40))).astype(np.int32) for _ in range(n // 3)]
    cands = [uniq[int(g.integers(len(uniq)))] for _ in range(n)]       # duplicate passages: exact ties
    flat, toff, seg, poff = build_pairs(2, 3, [(q, 8)] * 3, [[(d, len(d)) for d in cands]] * 2 + [[]], 512)
    pos, sc = enc.rerank(poff, flat, toff, seg, top_k)
    full = _all_scores(enc, flat, toff, seg, poff[:2], _native.RERANK_SIGMOID)
    order = np.lexsort((np.arange(n), -full))[:top_k]
    assert len(set(full.tolist())) < n                                 # there are ties
    for qi in range(2):
        assert pos[qi].tolist() == order.tolist()
        assert np.array_equal(sc[qi], full[order])
    assert (pos[2] == -1).all() and np.isnan(sc[2]).all()               # a query without candidates
    enc.destroy()


@pytest.mark.gpu
def test_rerank_leaves_the_embedding_path_alone(ctx):
    import bench
    from tests.test_gpu_embed import _embedder
    cfg = CE_MODELS["MiniLM-L6"]
    emb = _embedder(ctx, cfg, bench.random_bert_state(cfg, 3))
    toks = [np.random.default_rng(i).integers(1000, 30000, 20).astype(np.int32) for i in range(64)]
    before = [emb.embed(toks), emb.embed(toks)]
    enc = _encoder(ctx, cfg, _state(cfg, "bench"))
    flat, toff, seg, poff = _random_pairs(np.random.default_rng(1), 16, 30)
    enc.rerank(poff, flat, toff, seg, 5)
    after = emb.embed(toks)
    assert np.array_equal(before[0], after) and np.array_equal(before[1], after)
    enc.destroy(); emb.destroy()


@pytest.mark.gpu
def test_from_pretrained_and_store_retrieve(ctx, tmp_path):
    from kaito_b200.embedding import HashingEmbedding
    from kaito_b200.rerank import GpuCrossEncoder, build_pairs
    from kaito_b200.vector_store import VectorStore, embed_text
    from tests import st_snapshot as sts
    cfg = CE_MODELS["MiniLM-L6"]
    state = _state(cfg, "bench", seed=4)
    ce_cfg = dict(sts.MINILM_L6, architectures=["BertForSequenceClassification"], id2label={"0": "LABEL_0"}, label2id={"LABEL_0": 0})
    disk = {(k if k.startswith("classifier.") else "bert." + k): v for k, v in state.items()}
    sts.write(tmp_path, {"config.json": ce_cfg, "tokenizer_config.json": {"do_lower_case": True, "model_max_length": 512}}, state=disk)
    ce = GpuCrossEncoder.from_pretrained(ctx, str(tmp_path))
    assert ce.activation == "sigmoid" and ce.max_length == 512
    g = np.random.default_rng(2)
    words = [w for w in sts.VOCAB if not w.startswith("[") and not w.startswith("##")]
    docs = [{"text": " ".join(g.choice(words, int(g.integers(5, 60)))), "metadata": {"n": str(i % 3)}} for i in range(200)]
    plain = VectorStore(HashingEmbedding(384), ctx)
    rr = VectorStore(HashingEmbedding(384), ctx, reranker=ce)
    plain.index_documents("ce_plain", docs); rr.index_documents("ce_rr", docs)
    ref = br.Fp64CrossEncoder(cfg, state)
    for query in ("quick brown fox", "gpu token search passage"):
        got = rr.retrieve("ce_rr", query, max_node_count=10)
        fused = plain.retrieve("ce_plain", query, max_node_count=30)["results"]
        assert got["count"] == 10 and len(fused) == 30
        by_id = {n.node_id: n for n in plain.index_map["ce_plain"].nodes}
        texts = [embed_text(r["text"], by_id[r["node_id"]].metadata) for r in fused]
        q = ce.tokenizer.encode_batch_plain([query])[0]
        flat, toff, seg, _ = build_pairs(ce.tokenizer.cls, ce.tokenizer.sep, [(q, len(q))], [ce.encode_passages(texts)], 512)
        s64 = 1.0 / (1.0 + np.exp(-ref.logits(_pairs_of(flat, toff, seg, range(30)))[0]))
        want = np.lexsort((np.arange(30), -s64))[:10]
        ids = [r["node_id"] for r in got["results"]]
        for j, w in enumerate(want):
            if ids[j] != fused[w]["node_id"]:        # only a near-tie may swap
                other = [r["node_id"] for r in fused].index(ids[j])
                assert abs(s64[other] - s64[w]) < 2 * SCORE_TOL, (query, j)
        assert np.allclose([r["score"] for r in got["results"]], np.sort(s64)[::-1][:10], atol=SCORE_TOL)
