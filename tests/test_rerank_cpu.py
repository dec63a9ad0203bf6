"""CPU tests of cross-encoder reranking (kaito_b200.rerank): the snapshot reader and its refusals, the pair tokenisation
against transformers' BertTokenizer, and the store wiring of the three /retrieve paths with a numpy stand-in for the GPU
cross-encoder on the oracle engine."""
import json
import os

import numpy as np
import pytest

from kaito_b200.embedding import HashingEmbedding, load_state
from kaito_b200.rerank import build_pairs, check_head_tensors, pair_lengths, read_cross_encoder_spec
from kaito_b200.text import WordPieceTokenizer
from kaito_b200.vector_store import VectorStore, embed_text
from tests import st_snapshot as sts
from tests.test_wordpiece import VOCAB

MINILM_CE = dict(sts.MINILM_L6, architectures=["BertForSequenceClassification"], id2label={"0": "LABEL_0"},
                 label2id={"LABEL_0": 0}, sentence_transformers={"activation_fn": "torch.nn.modules.activation.Sigmoid"})
TOKENIZER_CONFIG = {"do_lower_case": True, "model_max_length": 512, "tokenizer_class": "BertTokenizer"}


def _snapshot(path, config=None, tokenizer_config=None):
    return sts.write(path, {"config.json": config or MINILM_CE, "tokenizer_config.json": tokenizer_config or TOKENIZER_CONFIG})


def test_minilm_cross_encoder_snapshot_is_accepted(tmp_path):
    spec = read_cross_encoder_spec(_snapshot(tmp_path))
    assert spec == {"max_length": 512, "do_lower_case": True, "activation": "sigmoid"}
    legacy = dict(MINILM_CE, sbert_ce_default_activation_function="torch.nn.modules.linear.Identity")
    del legacy["sentence_transformers"]
    assert read_cross_encoder_spec(_snapshot(tmp_path / "legacy", legacy))["activation"] == "identity"
    bare = {k: v for k, v in MINILM_CE.items() if k not in ("sentence_transformers", "id2label", "label2id")}
    bare["num_labels"] = 1
    spec = read_cross_encoder_spec(_snapshot(tmp_path / "bare", bare, {"model_max_length": int(1e30)}))
    assert spec == {"max_length": 512, "do_lower_case": True, "activation": "sigmoid"}


@pytest.mark.parametrize("change,file,field", [
    ({"id2label": {"0": "a", "1": "b"}}, "config.json", "2 labels"),
    ({"architectures": ["BertModel"]}, "config.json", "architectures"),
    ({"sentence_transformers": {"activation_fn": "torch.nn.modules.activation.Tanh"}}, "config.json", "Tanh"),
    ({"type_vocab_size": 1}, "config.json", "type_vocab_size"),
    ({"num_attention_heads": 8}, "config.json", "num_attention_heads 8"),        # 384 / 8 = head dim 48
    ({"max_position_embeddings": 256}, "tokenizer_config.json", "model_max_length 512"),
])
def test_refusals_name_the_file_and_field(tmp_path, change, file, field):
    with pytest.raises(ValueError) as e:
        read_cross_encoder_spec(_snapshot(tmp_path, dict(MINILM_CE, **change)))
    assert str(e.value).startswith(os.path.join(str(tmp_path), file) + ":") and field in str(e.value), str(e.value)


def test_missing_classifier_weight_is_refused(tmp_path):
    d = 128
    state = {"bert.embeddings.word_embeddings.weight": np.zeros((4, d)), "bert.pooler.dense.weight": np.zeros((d, d)),
             "bert.pooler.dense.bias": np.zeros(d), "classifier.bias": np.zeros(1)}
    sts.write(tmp_path, {"config.json": MINILM_CE}, state=state)
    with pytest.raises(ValueError) as e:
        check_head_tensors(str(tmp_path / "model.safetensors"), load_state(str(tmp_path)), d)
    assert str(e.value).startswith(str(tmp_path / "model.safetensors") + ":") and "classifier.weight" in str(e.value)
    state["classifier.weight"] = np.zeros((2, d))
    sts.write(tmp_path, {}, state=state)
    with pytest.raises(ValueError, match="classifier.weight has shape"):
        check_head_tensors("model.safetensors", load_state(str(tmp_path)), d)


# ------------------------------------------------------------------------------------------ pair tokenisation
PAIR_TEXTS = [("what is the quick fox", "The quick brown fox jumps over the lazy dog."),
              ("café naïvely", "中文 token, hello world"),
              ("gpu b200", ""),
              ("", "retrieval engine"),
              ("fox " * 20, "dog " * 20),                   # equal lengths at every cut
              ("fox " * 21, "dog " * 20),
              ("fox " * 20, "dog " * 23),
              ("fox " * 700, "the lazy dog"),               # a query longer than every max_length
              ("fox " * 600, "dog " * 700),
              ("fox " * 700, "dog " * 600),
              ("fox " * 260, "dog " * 255)]


@pytest.fixture(scope="module")
def vocab_file(tmp_path_factory):
    p = tmp_path_factory.mktemp("vocab") / "vocab.txt"
    seen, vocab = set(), []
    for t in VOCAB:
        if t not in seen:
            seen.add(t); vocab.append(t)
    p.write_text("\n".join(vocab) + "\n", encoding="utf-8")
    return str(p)


@pytest.mark.parametrize("m", [8, 16, 128, 512])
def test_pairs_match_transformers(vocab_file, m):
    transformers = pytest.importorskip("transformers")
    ref = transformers.BertTokenizer(vocab_file, do_lower_case=True)
    tok = WordPieceTokenizer.from_file(vocab_file, max_length=m)
    qs = [(q, len(q)) for q in tok.encode_batch_plain([q for q, _ in PAIR_TEXTS])]
    ds = [[(d[: m - 3], n)] for d, n in ((d, len(d)) for d in tok.encode_batch_plain([d for _, d in PAIR_TEXTS]))]
    flat, toff, seg, poff = build_pairs(tok.cls, tok.sep, qs, ds, m)
    assert poff.tolist() == list(range(len(PAIR_TEXTS) + 1))
    for i, (q, d) in enumerate(PAIR_TEXTS):
        # a batch of pairs, as sentence-transformers' CrossEncoder calls it (a lone empty text_pair would read as no pair)
        want = ref([q], [d], truncation="longest_first", max_length=m)
        got = flat[toff[i]:toff[i + 1]].tolist()
        assert got == want["input_ids"][0], (m, q[:20], d[:20])
        types = [0] * seg[i] + [1] * (len(got) - seg[i])
        assert types == want["token_type_ids"][0], (m, q[:20], d[:20])
    # the Python path of the tokeniser (non-ASCII or no native library) gives the same ids
    for (q, _), (qi, _) in zip(PAIR_TEXTS, qs):
        assert np.asarray([k for w in tok._basic(q) for k in tok._wordpiece(w)], np.int32).tolist() == qi.tolist()


def test_pair_lengths_rule():
    assert pair_lengths(3, 100, 13) == (3, 7)
    assert pair_lengths(100, 3, 13) == (7, 3)
    assert pair_lengths(10, 10, 13) == (5, 5)         # equal: budget 10 split evenly
    assert pair_lengths(10, 10, 14) == (5, 6)         # odd budget: the second half gets the extra token
    assert pair_lengths(11, 10, 14) == (6, 5)         # the longer half gets it
    assert pair_lengths(0, 50, 13) == (0, 10)
    assert pair_lengths(2, 3, 13) == (2, 3)


# ---------------------------------------------------------------------------------------------- store wiring
class FakeCrossEncoder:
    """GpuCrossEncoder's interface in numpy: score = shared words of query and passage / 4 (coarse, so ties are common),
    order = lexsort on (-score, fused position) -- the rule of krag_rerank"""

    def __init__(self):
        self.calls = []

    @staticmethod
    def encode_passages(texts):
        return [(set(t.lower().replace(".", " ").replace(":", " ").split()), len(t)) for t in texts]

    def score(self, query, words):
        return np.float32(len(set(query.lower().split()) & words) / 4.0)

    def rerank(self, queries, candidates, top_k, passages):
        self.calls.append([list(map(int, c)) for c in candidates])
        pos = np.full((len(queries), top_k), -1, np.int32)
        sc = np.full((len(queries), top_k), np.nan, np.float32)
        for i, (q, c) in enumerate(zip(queries, candidates)):
            s = np.array([self.score(q, w) for w, _ in passages(c, self.encode_passages)], np.float32)
            order = np.lexsort((np.arange(len(s)), -s))[:top_k]
            pos[i, :len(order)] = order
            sc[i, :len(order)] = s[order]
        return pos, sc


DOCS = [{"text": f"document {i} about " + " ".join(["gpu", "kernels", "fox", "dog", "retrieval", "cooking"][j] for j in range(i % 6 + 1)),
         "metadata": {"type": "even" if i % 2 == 0 else "odd"}} for i in range(40)]


def _stores(oracle, monkeypatch, **env):
    from tests.oracle_engine import OracleEngine
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    fake = FakeCrossEncoder()
    plain = VectorStore(HashingEmbedding(64), OracleEngine(oracle))
    rr = VectorStore(HashingEmbedding(64), OracleEngine(oracle), reranker=fake)
    for s in (plain, rr):
        s.index_documents("ix", DOCS)
    return plain, rr, fake


def _expected(plain, rr, fake, query, top_k, metadata_filter=None):
    """the reranked response computed from the plain store's fused list of N candidates"""
    n = min(max(top_k, rr.rerank_candidates), 300)
    fused = plain.retrieve("ix", query, max_node_count=n, metadata_filter=metadata_filter)["results"]
    st = rr.index_map["ix"]
    by_id = {nd.node_id: nd for nd in st.nodes}
    scores = [fake.score(query, fake.encode_passages([embed_text(r["text"], by_id[r["node_id"]].metadata)])[0][0]) for r in fused]
    order = sorted(range(len(fused)), key=lambda j: (-scores[j], j))[:top_k]
    return [(fused[j]["node_id"], float(scores[j])) for j in order], fused


@pytest.mark.parametrize("top_k", [1, 3, 10, 30, 45])
def test_rerank_order_and_scores(oracle, monkeypatch, top_k):
    plain, rr, fake = _stores(oracle, monkeypatch)
    for query in ("gpu kernels fox", "cooking dog retrieval gpu", "document"):
        want, fused = _expected(plain, rr, fake, query, top_k)
        got = rr.retrieve("ix", query, max_node_count=top_k)
        assert got["count"] == len(want) == min(top_k, len(fused))
        assert [(r["node_id"], r["score"]) for r in got["results"]] == want
        assert set(got["results"][0]) == {"doc_id", "node_id", "text", "score", "metadata"}
        assert len(fake.calls[-1][0]) == len(fused)         # N candidates went to the cross-encoder
    # the ties: many candidates share a score and keep their fused order among themselves
    want, _ = _expected(plain, rr, fake, "document", top_k)
    assert top_k < 3 or len({s for _, s in want}) < len(want)


def test_rerank_candidate_count(oracle, monkeypatch):
    plain, rr, fake = _stores(oracle, monkeypatch, KRAG_RERANK_CANDIDATES="12")
    rr.rerank_candidates = 12
    rr.retrieve("ix", "gpu fox", max_node_count=5)
    assert len(fake.calls[-1][0]) == 12
    rr.retrieve("ix", "gpu fox", max_node_count=20)              # top_k > candidates: N = top_k
    assert len(fake.calls[-1][0]) == 20
    small = VectorStore(HashingEmbedding(64), plain.engine.__class__(oracle), reranker=fake)
    small.index_documents("ix", DOCS[:4])                         # fewer fused candidates than N
    got = small.retrieve("ix", "gpu fox", max_node_count=10)
    assert got["count"] == 4 and len(fake.calls[-1][0]) == 4


def test_rerank_keyword_filter_and_paths_agree(oracle, monkeypatch):
    plain, rr, fake = _stores(oracle, monkeypatch)
    queries = ["gpu kernels fox", "cooking dog", "   ", "retrieval document"]
    for flt in (None, {"type": "even"}):
        for top_k in (1, 4, 30):
            dicts = rr.retrieve_batch("ix", queries, max_node_count=top_k, metadata_filter=flt)
            raw = rr.retrieve_batch_bytes("ix", queries, max_node_count=top_k, metadata_filter=flt)
            for q, d, b in zip(queries, dicts, raw):
                if not q.strip():
                    assert isinstance(d, Exception) and isinstance(b, Exception)
                    continue
                one = rr.retrieve("ix", q, max_node_count=top_k, metadata_filter=flt)
                assert d == one
                body, count, scores = b
                parsed = json.loads(body)
                for r in parsed["results"]:
                    assert r.pop("dense_score") is None and r.pop("sparse_score") is None and r.pop("source") is None
                assert parsed == d and count == d["count"] and scores == [r["score"] for r in d["results"]]
                want, _ = _expected(plain, rr, fake, q, top_k, flt)
                assert [(r["node_id"], r["score"]) for r in d["results"]] == want


def _with_components(store):
    """the oracle engine's retrieve plus per-result dense / sparse arrays (values derived from the ordinal, NaN = absent),
    as the fuse kernel returns them"""
    ix = store.index_map["ix"].index
    orig = ix.retrieve

    def retrieve(*a, **k):
        out = orig(*a, **k)
        o = np.asarray(out["ordinal"], np.float64)
        out["dense"] = np.where(o >= 0, o * 0.5, np.nan).astype(np.float32)
        out["sparse"] = np.where((o >= 0) & (o % 3 != 0), o + 0.25, np.nan).astype(np.float32)
        return out
    ix.retrieve = retrieve


def test_rerank_component_scores_describe_the_fusion(oracle, monkeypatch):
    plain, rr, fake = _stores(oracle, monkeypatch, KRAG_COMPONENT_SCORES="1")
    assert rr.component_scores and plain.component_scores
    _with_components(plain); _with_components(rr)
    q = "gpu kernels fox"
    fused = plain.retrieve("ix", q, max_node_count=30)["results"]
    comp = {r["node_id"]: (r["dense_score"], r["sparse_score"], r["source"]) for r in fused}
    for got in (rr.retrieve("ix", q, max_node_count=7), rr.retrieve_batch("ix", [q], max_node_count=7)[0],
                json.loads(rr.retrieve_batch_bytes("ix", [q], max_node_count=7)[0][0])):
        assert got["count"] == 7
        for r in got["results"]:
            assert (r["dense_score"], r["sparse_score"], r["source"]) == comp[r["node_id"]]


def test_pair_cache_is_filled_once_and_cleared_by_compaction(oracle, monkeypatch):
    plain, rr, fake = _stores(oracle, monkeypatch)
    st = rr.index_map["ix"]
    rr.retrieve("ix", "gpu fox", max_node_count=5)
    assert len(st._pair_cache) == 30
    seen = []
    cached = sorted(st._pair_cache)[:2]
    st.pair_passages(cached, lambda texts: seen.append(texts) or fake.encode_passages(texts))
    assert seen == []                                        # hits: no tokenisation
    st.n_dead = 10 ** 6                                      # past both compaction thresholds
    st.index.compact = lambda: None                          # the engine side of the compaction is not under test here
    rr._maybe_compact(st)
    assert st._pair_cache == {}
