"""GPU tests of late-interaction (ColBERT) reranking: krag_late_rerank and krag_debug_late_vectors against an fp64
transformers.BertModel run with ColBERT's attention mask, the projection, the normalisation and MaxSim in fp64
(tests/colbert_reference.py).  Token vectors and scores are held to F = 40 times torch fp32's own error against fp64, as the
K5 tests are; the fp16 mode to torch bf16 autocast's error.  Random weights (no checkpoints offline)."""
import numpy as np
import pytest

from tests import bert_reference as br
from tests import colbert_reference as cr

F = 40.0
QL = 32
SHAPES = {   # the encoder and projection of colbert-ir/colbertv2.0 and answerdotai/answerai-colbert-small-v1
    "colbertv2.0": (dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=30522,
                         max_position_embeddings=512), 128),
    "answerai-colbert-small": (dict(num_hidden_layers=12, hidden_size=384, num_attention_heads=12, intermediate_size=1536,
                                    vocab_size=30522, max_position_embeddings=512), 96),
}


def _state(cfg, dim, regime, seed=0):
    import bench
    if regime == "stressed":
        cfg = dict(cfg, num_hidden_layers=2)          # stressed weights run on 2 layers (see DESIGN.md, K5 bounds)
        st = br.stressed_state(cfg, seed)[0]
    else:
        st = bench.random_bert_state(cfg, seed)
    w = (np.random.default_rng(seed + 9).standard_normal((dim, cfg["hidden_size"])) / np.sqrt(cfg["hidden_size"])).astype(np.float32)
    return cfg, st, w


def _model(ctx, cfg, st, w, precision="fp32"):
    from kaito_b200 import _native
    e = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                         cfg["vocab_size"], cfg["max_position_embeddings"])
    e.set_late_interaction(w)
    e.load_state_dict(st)
    e.set_precision(precision)
    return e


def _query(g, n_real):
    ids = np.full(QL, 103, np.int32)                  # [MASK]
    n = min(n_real, QL - 3) + 3
    ids[0], ids[1], ids[n - 1] = 101, 1, 102          # [CLS] [unused0] ... [SEP]
    ids[2:n - 1] = g.integers(1000, 30000, n - 3)
    return ids, n


def _passage(g, n):
    ids = np.concatenate([[101, 2], g.integers(1000, 30000, n), [102]]).astype(np.int32)
    keep = (g.random(len(ids)) > 0.15).astype(np.uint8)
    keep[0] = 1
    return ids, keep


def _all_scores(e, qs, qk, docs, cands, top_k=None):
    """every pair's score in pair order (put back by position; NaN where top_k leaves a pair out) and the selection"""
    d_off = np.concatenate([[0], np.cumsum([len(d[0]) for d in docs])]).astype(np.int32)
    poff = np.concatenate([[0], np.cumsum([len(c) for c in cands])]).astype(np.int32)
    pp = np.concatenate([np.asarray(c, np.int32) for c in cands])
    k = top_k or int(np.diff(poff).max())
    pos, sc = e.late_rerank(np.stack(qs), qk, np.concatenate([d[0] for d in docs]), d_off, np.concatenate([d[1] for d in docs]),
                            poff, pp, k)
    out = np.full(int(poff[-1]), np.nan, np.float32)
    for q in range(len(cands)):
        n = min(len(cands[q]), k)
        out[poff[q] + pos[q, :n]] = sc[q, :n]
    return out, pos, sc


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["bench", "stressed"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_vectors_and_scores_match_fp64(ctx, shape, regime):
    cfg, st, w = _state(*SHAPES[shape], regime)
    e = _model(ctx, cfg, st, w)
    ref = cr.Fp64ColBERT(cfg, st, w)
    g = np.random.default_rng(3)
    qs, qk = zip(*[_query(g, n) for n in (0, 5, 29, 40)])          # empty, short, exactly full, over-long queries
    docs = [_passage(g, n) for n in (0, 10, 125, 177, 60, 177)]
    cands = [[0, 1, 2], [3, 4, 5], [5, 1], [2, 3, 4, 0]]
    got, _, _ = _all_scores(e, qs, np.asarray(qk), docs, cands)
    v_err = t_err = s_err = s32_err = 0.0
    q64, q32 = zip(*[ref.vectors(q, k) for q, k in zip(qs, qk)])
    d64, d32 = zip(*[ref.vectors(d[0]) for d in docs])
    gq = e.debug_late_vectors(np.concatenate(qs), np.arange(0, QL * len(qs) + 1, QL), np.asarray(qk)).reshape(len(qs), QL, -1)
    for i in range(len(qs)):
        v_err = max(v_err, float(np.abs(gq[i] - q64[i]).max())); t_err = max(t_err, float(np.abs(q32[i] - q64[i]).max()))
    p = 0
    for q, c in enumerate(cands):
        for j in c:
            s64 = cr.maxsim(q64[q], d64[j], docs[j][1])
            s_err = max(s_err, abs(float(got[p]) - s64))
            s32_err = max(s32_err, abs(cr.maxsim(q32[q], d32[j], docs[j][1]) - s64))
            p += 1
    vr, sr = v_err / max(t_err, 2.0 ** -23), s_err / max(s32_err, 2.0 ** -23)
    print(f"colbert vs fp64 | {shape} {regime} | vector err {v_err:.2e} (torch fp32 {t_err:.2e}, ratio {vr:.2f}) | "
          f"score err {s_err:.2e} (torch fp32 {s32_err:.2e}, ratio {sr:.2f})")
    assert vr <= F and sr <= F, (vr, sr)
    e.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
def test_fp16_mode_within_bf16_autocast_error(ctx, shape):
    cfg, st, w = _state(*SHAPES[shape], "bench")
    e = _model(ctx, cfg, st, w, precision="fp16")
    ref = cr.Fp64ColBERT(cfg, st, w)
    g = np.random.default_rng(4)
    qs, qk = zip(*[_query(g, n) for n in (3, 12)])
    docs = [_passage(g, n) for n in (40, 177, 90)]
    cands = [[0, 1, 2], [2, 1, 0]]
    got, _, _ = _all_scores(e, qs, np.asarray(qk), docs, cands)
    k5 = bf = 0.0
    p = 0
    for q, c in enumerate(cands):
        q64 = ref.vectors(qs[q], qk[q])[0]; qb = ref.vectors_bf16(qs[q], qk[q])
        for j in c:
            s64 = cr.maxsim(q64, ref.vectors(docs[j][0])[0], docs[j][1])
            k5 = max(k5, abs(float(got[p]) - s64)); bf = max(bf, abs(cr.maxsim(qb, ref.vectors_bf16(docs[j][0]), docs[j][1]) - s64))
            p += 1
    print(f"colbert fp16 | {shape} | score err {k5:.2e} | torch bf16 autocast {bf:.2e} | ratio {k5 / bf:.2f}")
    assert k5 <= bf, (k5, bf)
    e.destroy()


@pytest.mark.gpu
def test_mask_rows_are_not_keys(ctx):
    """attend_to_mask_tokens false: a query's real rows are the bits of a forward without its [MASK] rows; true: the [MASK]
    rows are keys (the real rows move) and match fp64"""
    cfg, st, w = _state(*SHAPES["answerai-colbert-small"], "bench", seed=1)
    e = _model(ctx, cfg, st, w)
    ref = cr.Fp64ColBERT(cfg, st, w)
    g = np.random.default_rng(6)
    q, n = _query(g, 9)
    padded = e.debug_late_vectors(q, np.array([0, QL]), np.array([n]))
    alone = e.debug_late_vectors(q[:n], np.array([0, n]))
    assert np.array_equal(padded[:n], alone)
    full = e.debug_late_vectors(q, np.array([0, QL]), np.array([QL]))
    assert np.array_equal(full, e.debug_late_vectors(q, np.array([0, QL])))      # key length = length: no key lengths
    assert not np.array_equal(full[:n], padded[:n])
    for keys, got in ((n, padded), (QL, full)):
        v64, v32 = ref.vectors(q, keys)
        assert float(np.abs(got - v64).max()) <= F * max(float(np.abs(v32 - v64).max()), 2.0 ** -23)
    e.destroy()


@pytest.mark.gpu
def test_ragged_ties_and_dedupe(ctx):
    cfg, st, w = _state(*SHAPES["answerai-colbert-small"], "bench", seed=2)
    e = _model(ctx, cfg, st, w)
    g = np.random.default_rng(8)
    qs, qk = zip(*[_query(g, n) for n in (4, 7, 11)])
    docs = [_passage(g, n) for n in (30, 70, 150, 20)]
    # passage 1 twice within query 0 (equal scores: the lower position wins), passages shared across queries, a query with
    # fewer candidates than top_k and one with none
    cands = [[1, 0, 1, 2, 3], [3, 2], []]
    dedup, _, _ = _all_scores(e, qs, np.asarray(qk), docs, cands)
    _, pos, sc = _all_scores(e, qs, np.asarray(qk), docs, [cands[0][:4], cands[1], []], top_k=4)
    assert np.array_equal(sc[0], np.sort(dedup[:4])[::-1])
    _, pos, sc = _all_scores(e, qs, np.asarray(qk), docs, cands, top_k=4)
    assert pos[0].tolist() == [int(x) for x in np.lexsort((np.arange(5), -dedup[:5]))[:4]]
    assert dedup[0] == dedup[2]
    assert pos[1, 2:].tolist() == [-1, -1] and np.isnan(sc[1, 2:]).all()
    assert (pos[2] == -1).all() and np.isnan(sc[2]).all()
    # no dedupe: every pair its own copy of its passage
    flat = [docs[j] for c in cands for j in c]
    own = [list(range(0, 5)), [5, 6], []]
    sep, _, _ = _all_scores(e, qs, np.asarray(qk), flat, own)
    assert np.array_equal(dedup, sep)
    # a pair's score does not depend on the other pairs of the call
    alone, _, _ = _all_scores(e, qs[1:2], np.asarray(qk[1:2]), [docs[2]], [[0]])
    assert alone[0] == dedup[6]
    e.destroy()


@pytest.mark.gpu
def test_from_pretrained_and_store_retrieve(ctx, tmp_path):
    import json
    from kaito_b200.embedding import HashingEmbedding
    from kaito_b200.rerank import GpuLateInteractionReranker
    from kaito_b200.vector_store import VectorStore, embed_text
    from tests import st_snapshot as sts
    vocab = sts.VOCAB + ["[unused0]", "[unused1]"]
    base = dict(SHAPES["answerai-colbert-small"][0], num_hidden_layers=4, vocab_size=len(vocab))
    cfg, st, w = _state(base, 96, "bench", seed=5)
    disk = {"bert." + k: v for k, v in st.items()}
    disk["linear.weight"] = w
    sts.write(tmp_path, {"config.json": dict(sts.BGE_SMALL, **base, architectures=["HF_ColBERT"]),
                         "tokenizer_config.json": {"do_lower_case": True}}, vocab=vocab, state=disk)
    with open(tmp_path / "artifact.metadata", "w") as f:
        json.dump({"query_maxlen": 32, "doc_maxlen": 180, "dim": 96, "mask_punctuation": True, "attend_to_mask_tokens": False,
                   "query_token_id": "[unused0]", "doc_token_id": "[unused1]", "similarity": "cosine"}, f)
    rr_model = GpuLateInteractionReranker.from_pretrained(ctx, str(tmp_path))
    ref = cr.Fp64ColBERT(cfg, st, w)
    g = np.random.default_rng(2)
    words = [x for x in sts.VOCAB if not x.startswith("[") and not x.startswith("##")]
    docs = [{"text": " ".join(g.choice(words, int(g.integers(5, 60)))), "metadata": {"n": str(i % 3)}} for i in range(200)]
    plain = VectorStore(HashingEmbedding(384), ctx)
    rr = VectorStore(HashingEmbedding(384), ctx, reranker=rr_model)
    plain.index_documents("cb_plain", docs); rr.index_documents("cb_rr", docs)
    for query in ("quick brown fox", "gpu token search passage"):
        got = rr.retrieve("cb_rr", query, max_node_count=10)
        fused = plain.retrieve("cb_plain", query, max_node_count=30)["results"]
        by_id = {nd.node_id: nd for nd in plain.index_map["cb_plain"].nodes}
        ps = rr_model.encode_passages([embed_text(r["text"], by_id[r["node_id"]].metadata) for r in fused])
        qi, qk = rr_model.query_ids([query])
        q64, q32 = ref.vectors(qi[0], qk[0])
        s64, s32 = [], []
        for ids, keep in ps:
            d64, d32 = ref.vectors(ids)
            s64.append(cr.maxsim(q64, d64, keep)); s32.append(cr.maxsim(q32, d32, keep))
        s64 = np.asarray(s64)
        bound = F * max(float(np.abs(np.asarray(s32) - s64).max()), 2.0 ** -23)
        want = np.lexsort((np.arange(30), -s64))[:10]
        ids = [r["node_id"] for r in got["results"]]
        fused_ids = [r["node_id"] for r in fused]
        for j, wj in enumerate(want):
            if ids[j] != fused[wj]["node_id"]:                       # only scores within twice the bound may swap
                assert abs(s64[fused_ids.index(ids[j])] - s64[wj]) <= 2 * bound, (query, j)
        assert np.allclose([r["score"] for r in got["results"]], np.sort(s64)[::-1][:10], atol=bound)
    rr_model._emb.destroy()


@pytest.mark.gpu
def test_fp16_scores_do_not_depend_on_the_call_size(ctx):
    """fp16 mode: a pair's score has the same bits in a call of 40 passages (over 7,000 tokens: enough 128-row tiles that
    the general GEMM plan would take 128 x 256 tiles at the colbertv2.0 shape) as in a call of its own"""
    cfg, st, w = _state(dict(SHAPES["colbertv2.0"][0], num_hidden_layers=2), 128, "bench", seed=3)
    e = _model(ctx, cfg, st, w, precision="fp16")
    g = np.random.default_rng(12)
    q, n = _query(g, 10)
    docs = [_passage(g, 177) for _ in range(40)]
    many, _, _ = _all_scores(e, [q], np.array([n]), docs, [list(range(40))])
    for j in (0, 17, 39):
        alone, _, _ = _all_scores(e, [q], np.array([n]), [docs[j]], [[0]])
        assert alone[0] == many[j], j
    e.destroy()


@pytest.mark.gpu
def test_refusals(ctx):
    from kaito_b200 import _native
    cfg, st, w = _state(dict(SHAPES["answerai-colbert-small"][0], num_hidden_layers=1), 96, "bench", seed=4)
    e = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                         cfg["vocab_size"], cfg["max_position_embeddings"])
    with pytest.raises(_native.KragError, match="linear.weight") as ex:
        e.set_late_interaction(w[:, :-16])                                # [96, 368]: not dim x hidden
    assert ex.value.code == _native.KRAG_E_INVALID
    e.destroy()
    e = _model(ctx, cfg, st, w)
    g = np.random.default_rng(1)
    q, n = _query(g, 5)
    ids, keep = _passage(g, 20)
    args = lambda qk=n, kp=keep, pp=(0,): (q[None], np.array([qk]), ids, np.array([0, len(ids)]), kp, np.array([0, len(pp)]),  # noqa: E731
                                           np.array(pp), 1)
    e.late_rerank(*args())                                                # the valid call
    for bad, what in ((args(qk=0), "key length"), (args(qk=QL + 1), "key length"), (args(kp=np.zeros_like(keep)), "at least one row"),
                      (args(pp=(1,)), "passage index"), (args(pp=(-1,)), "passage index")):
        with pytest.raises(_native.KragError, match=what) as ex:
            e.late_rerank(*bad)
        assert ex.value.code == _native.KRAG_E_INVALID
    e.destroy()
