"""CPU tests: the oracle against the reference-generated golden fixtures and against
independent restatements.  No GPU, no reference checkout at run time."""
import json
import math
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden", "fuse_reference.json")


@pytest.fixture(scope="module")
def gold():
    with open(GOLD) as f:
        return json.load(f)


def _tie_groups_equal(ids_a, fin_a, ids_b, fin_b):
    """same finals position by position; ids equal as sets inside runs of equal finals"""
    assert list(fin_a) == list(fin_b)
    i = 0
    while i < len(fin_a):
        j = i
        while j < len(fin_a) and fin_a[j] == fin_a[i]:
            j += 1
        assert sorted(ids_a[i:j]) == sorted(ids_b[i:j])
        i = j


def test_pool_and_weights_match_reference_constructor(oracle, gold):
    for c in gold["init"]:
        assert oracle.pool_size(c["max_results"], c["candidate_multiplier"]) == c["pool"]
        total = c["vector_weight"] + c["text_weight"]
        assert c["vector_weight"] / total == c["w_v"] and c["text_weight"] / total == c["w_t"]


def test_c_fuse_matches_reference_fuse(oracle, gold):
    for c in gold["fuse"]:
        fin, de, sp, rk, od = oracle.fuse(np.array(c["dense_dist"], np.float32), np.array(c["dense_ids"], np.int64),
                                          np.array(c["bm25_score"], np.float32), np.array(c["bm25_ids"], np.int64),
                                          c["k"], c["vector_weight"], c["text_weight"])
        # the reference may cut a tie group at k differently: compare the common guaranteed part
        ref_ids, ref_fin = c["out_ids"], c["out_final"]
        assert len(od) == len(ref_ids)
        if len(ref_fin) and ref_fin.count(ref_fin[-1]) > 0:
            # drop a trailing tie group that might be truncated by [:k]
            last = ref_fin[-1]
            cut = len(ref_fin)
            all_final = sorted([f for f in _all_finals(c)], reverse=True)
            if all_final.count(last) > ref_fin.count(last):
                cut = ref_fin.index(last)
            _tie_groups_equal(list(od[:cut]), list(fin[:cut]), ref_ids[:cut], ref_fin[:cut])
            assert list(fin) == ref_fin


def _all_finals(c):
    total = c["vector_weight"] + c["text_weight"]
    wv, wt = c["vector_weight"] / total, c["text_weight"] / total
    vs = dict(zip(c["dense_ids"], c["dense_dist"]))
    kr = {i: r for r, i in enumerate(c["bm25_ids"])}
    for nid in set(vs) | set(kr):
        yield wv * vs.get(nid, 0.0) + wt * (1.0 / (1.0 + kr[nid]) if nid in kr else 0.0)


def test_py_fuse_matches_reference_fuse(oracle, gold):
    for c in gold["fuse"]:
        out = oracle.py_fuse(list(zip(c["dense_ids"], c["dense_dist"])), list(zip(c["bm25_ids"], c["bm25_score"])),
                             c["k"], c["vector_weight"], c["text_weight"])
        assert [f for _, f in out] == c["out_final"]


def test_retrieve_flow_with_keyword_post_filter(oracle, gold):
    for c in gold["retrieve_flow"]:
        k = c["k"]
        P = oracle.pool_size(k)
        assert c["seen_top_k"] == P
        dense = c["dense"][:P]
        kw = c["keyword"][:P]
        if c["metadata_filter"]:
            kw = [x for x in kw if x[2] == c["metadata_filter"]["tag"]]
        fin, de, sp, rk, od = oracle.fuse(np.array([x[1] for x in dense], np.float32), np.array([x[0] for x in dense], np.int64),
                                          np.array([x[1] for x in kw], np.float32), np.array([x[0] for x in kw], np.int64), k)
        assert list(fin) == c["out_final"]
        assert sorted(od.tolist()) == sorted(c["out_ids"]) or len(set(c["out_final"])) < len(c["out_final"])


def test_vector_only_fallback(gold):
    c = gold["vector_only_fallback"]
    assert c["out_ids"] == [x[0] for x in c["dense"][: c["k"]]]


def test_l2sq_close_to_fp64_and_order_defined(oracle):
    for d in (8, 33, 384, 768, 1000, 1024):
        x = oracle.synth_dense(257, d, seed=d)
        q = oracle.synth_queries(x, 3, seed=d + 1)
        for b in range(3):
            got = oracle.l2sq(x, q[b])
            ref = oracle.np_l2sq_f64(x, q[b])
            assert np.max(np.abs(got - ref)) < 2e-6
    # the documented summation order, restated in numpy for d = 64
    x = oracle.synth_dense(5, 64, 7)
    q = oracle.synth_queries(x, 1, 8)[0]
    for r in range(5):
        p = np.zeros(32, np.float32)
        for i in range(64):
            t = np.float32(x[r, i] - q[i])
            p[i % 32] = np.float32(math.fma(float(t), float(t), float(p[i % 32]))) if hasattr(math, "fma") else np.float32(np.float64(t) * np.float64(t) + np.float64(p[i % 32]))
        s = [np.float32(np.float32(p[4 * l] + p[4 * l + 1]) + np.float32(p[4 * l + 2] + p[4 * l + 3])) for l in range(8)]
        a = [np.float32(s[i] + s[i + 4]) for i in range(4)]
        res = np.float32(np.float32(a[0] + a[2]) + np.float32(a[1] + a[3]))
        assert res == oracle.l2sq(x[r:r + 1], q)[0]


def test_dense_topk_matches_argsort(oracle):
    x = oracle.synth_dense(5000, 96, 1)
    q, rows = oracle.synth_queries(x, 6, 2, return_rows=True)
    dist, ordn = oracle.dense_topk(x, q, 30)
    for b in range(6):
        d = oracle.l2sq(x, q[b])
        order = np.lexsort((np.arange(len(d)), d))[:30]
        assert ordn[b].tolist() == order.tolist()
        assert np.array_equal(dist[b], d[order])
    # planted neighbours come back first
    assert ordn[0, 0] == rows[0] and ordn[1, 0] == rows[1] and ordn[2, 0] == rows[2]
    # tombstones + short corpus
    alive = oracle.alive_bitmap(5000, dead=ordn[0, :5].tolist())
    dist2, ord2 = oracle.dense_topk(x, q[:1], 30, alive)
    assert not set(ordn[0, :5].tolist()) & set(ord2[0].tolist())
    dist3, ord3 = oracle.dense_topk(x[:7], q[:1], 30)
    assert (ord3[0, 7:] == -1).all() and np.isinf(dist3[0, 7:]).all() and (ord3[0, :7] >= 0).all()


def test_dense_topk_against_third_party_brute_force(oracle):
    """faiss is not installable here (DESIGN.md section 2), but two other exact L2 searches are: scikit-learn's brute-force
    NearestNeighbors and scipy's cdist.  The oracle's top-P must be theirs -- same ids in the same order wherever the fp64
    distances are further apart than fp32 rounding, squared distances within 2e-6."""
    sk = pytest.importorskip("sklearn.neighbors")
    sp = pytest.importorskip("scipy.spatial.distance")
    for n, d, P in ((4000, 384, 30), (2500, 768, 90), (1500, 1024, 30)):
        x = oracle.synth_dense(n, d, seed=n)
        q = oracle.synth_queries(x, 5, seed=d)
        dist, ordn = oracle.dense_topk(x, q, P)
        nn = sk.NearestNeighbors(n_neighbors=P, algorithm="brute", metric="sqeuclidean").fit(x.astype(np.float64))
        ref_d, ref_i = nn.kneighbors(q.astype(np.float64))
        full = sp.cdist(q.astype(np.float64), x.astype(np.float64), "sqeuclidean")
        for b in range(len(q)):
            assert np.max(np.abs(dist[b] - ref_d[b])) < 2e-6
            assert np.max(np.abs(dist[b] - full[b, ordn[b]])) < 2e-6
            for j in np.nonzero(ordn[b] != ref_i[b])[0]:          # order may differ only between near-ties
                assert abs(full[b, ordn[b, j]] - full[b, ref_i[b, j]]) < 2e-6
            assert set(ordn[b].tolist()) == set(ref_i[b].tolist()) or \
                np.max(np.abs(np.sort(full[b, ordn[b]]) - np.sort(full[b, ref_i[b]]))) < 2e-6


def test_bm25_scores_match_python_restatement(oracle):
    off, ids, tf, dl = oracle.synth_sparse(300, 500, seed=3)
    post = oracle.bm25_build(off, ids, tf, dl, 500)
    df = oracle.bm25_df(off, ids, 500)
    avgdl = float(dl.astype(np.int64).sum()) / 300
    # every posting equals the line-by-line Python formula
    tf_of = {}
    for d in range(300):
        for i in range(off[d], off[d + 1]):
            tf_of[(int(ids[i]), d)] = int(tf[i])
    for t in range(500):
        docs = post.doc[post.off[t]:post.off[t + 1]]
        assert (np.diff(docs.astype(np.int64)) > 0).all()  # ascending inside a term
        assert len(docs) == df[t]
        for p in range(post.off[t], post.off[t + 1]):
            d = int(post.doc[p])
            assert post.score[p] == oracle.py_bm25_score(int(df[t]), 300, tf_of[(t, d)], int(dl[d]), avgdl)


def test_bm25_query_semantics(oracle):
    off, ids, tf, dl = oracle.synth_sparse(400, 300, seed=5)
    post = oracle.bm25_build(off, ids, tf, dl, 300)
    qs = oracle.synth_query_terms(300, 5, seed=6, rank_offset=3)
    for qt in qs:
        qt = np.concatenate([qt, qt[:1]])  # a duplicated term counts twice (bm25s sums per token)
        score, ordn = oracle.bm25_query(post, qt, 30)
        acc = np.zeros(400, np.float32)
        for t in qt:
            sl = slice(post.off[t], post.off[t + 1])
            acc[post.doc[sl]] += post.score[sl]
        order = np.lexsort((np.arange(400), -acc.astype(np.float64)))[:30]
        assert ordn.tolist() == order.tolist()
        assert np.array_equal(score, acc[order])
    # zero-score fill: a term nobody has -> lowest ordinals, score 0; P clamps to N
    score, ordn = oracle.bm25_query(oracle.bm25_build(off[:6], ids[:off[5]], tf[:off[5]], dl[:5], 300),
                                    np.array([299], np.uint32), 8)
    assert ordn.tolist()[:5] == [0, 1, 2, 3, 4] and ordn.tolist()[5:] == [-1, -1, -1]


def test_doc_id_is_sha256_hex(oracle):
    # reference: tests/api/test_main.py:28,45 and vector_store/base.py:82-85
    h = oracle.generate_doc_id("This is a test document")
    assert len(h) == 64 and int(h, 16) >= 0
    import hashlib
    assert h == hashlib.sha256(b"This is a test document").hexdigest()


# ------------------------------------------------------------------ third-party pins (present only where the wheels exist)
GOLD_3P = os.path.join(os.path.dirname(__file__), "golden", "third_party_reference.json")


@pytest.mark.skipif(not os.path.exists(GOLD_3P), reason="tests/golden/third_party_reference.json not generated: faiss / bm25s / "
                    "PyStemmer are not installable offline (run oracle/gen_golden_3p.py where they are)")
def test_third_party_golden(oracle):
    """the oracle's restated dense L2^2, BM25 (bm25s lucene) and Snowball stems against outputs of the REAL wheels"""
    from kaito_b200 import text as T
    doc = json.load(open(GOLD_3P))
    sec = doc["sections"]
    if "pystemmer_english" in sec:
        s = sec["pystemmer_english"]
        assert [T.stem(w) for w in s["words"]] == s["stems"]
    if "faiss_flat_l2" in sec:
        for c in sec["faiss_flat_l2"]["cases"]:
            if c["x"] is None:
                continue
            x, q = np.array(c["x"], np.float32), np.array(c["q"], np.float32)
            k = min(c["k"], c["n"])
            dist, ids = oracle.dense_topk(x, q, k)
            want_d, want_i = np.array(c["dist"], np.float32)[:, :k], np.array(c["ids"], np.int64)[:, :k]
            assert np.allclose(dist, want_d, atol=1e-4, rtol=0)            # north_star: scores within 1e-4 fp32
            # ids equal wherever faiss' own ordering is unambiguous (gap to the neighbours above the fp32 noise)
            gap = np.minimum(np.abs(np.diff(want_d, axis=1, prepend=-1)), np.abs(np.diff(want_d, axis=1, append=9)))
            assert np.array_equal(ids[gap > 1e-5], want_i[gap > 1e-5])
    if "bm25s_lucene" in sec:
        b = sec["bm25s_lucene"]
        n, vocab = len(b["corpus_token_ids"]), len(b["vocab"])
        off, ids, tf, dl = [0], [], [], []
        for toks in b["corpus_token_ids"]:
            u, cnt = np.unique(np.array(toks, np.int64), return_counts=True)
            ids += u.tolist(); tf += cnt.tolist(); off.append(len(ids)); dl.append(len(toks))
        post = oracle.bm25_build(np.array(off, np.int64), np.array(ids, np.uint32), np.array(tf, np.uint16), np.array(dl, np.uint32), vocab)
        for qq in b["queries"]:
            qt = np.array([b["vocab"][t] for t in qq["query_tokens"] if t in b["vocab"]], np.uint32)
            rs, ro = oracle.bm25_query(post, qt, n)
            want = dict(zip(qq["doc_ids"], qq["scores"]))
            for o, s in zip(ro, rs):
                assert np.float32(want[int(o)]) == np.float32(s), (qq["query"], int(o))     # same fp32 score per document
