"""CPU tests of the ColBERT passage vector store's host side: which ordinals the service appends with which texts, the
rollback when the engine's add fails, the compaction bitmap against the host's renumbering, the rebuild at /load, the
reranker seeing the index's store, and the start-up refusals of KRAG_RERANK_STORE_GB.  A recording store and reranker
stand in for the GPU (kaito_b200.rerank.PassageStore / GpuLateInteractionReranker), an oracle engine for the index."""
import numpy as np
import pytest

from kaito_b200 import _native, rerank
from kaito_b200 import vector_store as vs
from kaito_b200.embedding import HashingEmbedding
from tests import st_snapshot as sts
from tests.test_compact_cpu import WORDS, CompactingOracleEngine
from tests.test_rerank_cpu import MINILM_CE, TOKENIZER_CONFIG


class FakeStore:
    """PassageStore's interface over a list: entry o is the text appended for ordinal o"""

    def __init__(self):
        self.texts, self.calls, self.destroyed = [], [], False

    def __len__(self):
        return len(self.texts)

    def append(self, texts):
        self.calls.append(("append", len(self.texts), list(texts)))
        self.texts.extend(texts)

    def truncate(self, n):
        self.calls.append(("truncate", n))
        del self.texts[n:]

    def compact(self, alive):
        alive = list(alive)
        assert len(alive) == len(self.texts)
        self.calls.append(("compact", alive))
        self.texts = [t for t, a in zip(self.texts, alive) if a]

    def destroy(self):
        self.destroyed = True


class FakeReranker:
    """ranks candidates in fused order; records the store each call saw"""

    def __init__(self):
        self.stores, self.seen = [], []

    def create_store(self):
        self.stores.append(FakeStore())
        return self.stores[-1]

    def encode_passages(self, texts):
        return [(np.zeros(3, np.int32), np.ones(3, np.uint8)) for _ in texts]

    def rerank(self, queries, candidates, top_k, passages, store=None):
        self.seen.append(store)
        pos = np.full((len(queries), top_k), -1, np.int32)
        sc = np.full((len(queries), top_k), np.nan, np.float32)
        for q, c in enumerate(candidates):
            n = min(len(c), top_k)
            pos[q, :n] = np.arange(n)
            sc[q, :n] = -np.arange(n, dtype=np.float32)
        return pos, sc


def _docs(n, seed):
    rng = np.random.default_rng(seed)
    return [{"text": f"doc {seed}-{i}: " + " ".join(rng.choice(WORDS, size=int(rng.integers(4, 12)))),
             "metadata": {"tag": "a" if i % 3 else "b"}} for i in range(n)]


def _store(oracle):
    rr = FakeReranker()
    return vs.VectorStore(HashingEmbedding(64), CompactingOracleEngine(oracle), reranker=rr), rr


def _texts(st):
    return [vs.embed_text(n.text, n.metadata) for n in st.nodes]


def test_index_appends_every_new_ordinal_with_its_embed_text(oracle):
    store, rr = _store(oracle)
    store.index_documents("ix", _docs(20, 1))
    store.index_documents("ix", _docs(20, 1) + _docs(5, 2))          # the repeats are skipped: only 5 new documents
    st = store.index_map["ix"]
    fake = st.late_store
    assert rr.stores == [fake]
    assert fake.texts == _texts(st)
    assert [c[1] for c in fake.calls] == [0, 20]                      # each append starts at the ordinal count before it
    store.retrieve("ix", "retrieval engine", max_node_count=3)
    assert rr.seen[-1] is fake


def test_a_failing_add_rolls_the_store_back(oracle):
    store, _ = _store(oracle)
    store.index_documents("ix", _docs(10, 1))
    st = store.index_map["ix"]

    def broken(*a, **k):
        raise RuntimeError("engine add failed")
    st.index.add = broken
    with pytest.raises(RuntimeError, match="engine add failed"):
        store.index_documents("ix", _docs(4, 3))
    assert st.late_store.calls[-1] == ("truncate", 10)
    assert len(st.late_store) == 10 and st.late_store.texts == _texts(st)


@pytest.mark.parametrize("renumbers", [False, True])
def test_compaction_keeps_the_store_aligned_with_the_renumbered_nodes(oracle, monkeypatch, renumbers):
    monkeypatch.setattr(vs, "COMPACT_MIN_DEAD_ROWS", 4)
    monkeypatch.setattr(vs, "COMPACT_DEAD_FRACTION", 0.25)
    store, _ = _store(oracle)
    docs = _docs(30, 4)
    ids = store.index_documents("ix", docs)
    st = store.index_map["ix"]
    st.index.compact_renumbers_keys = renumbers
    if renumbers:                                                     # the sharded engine's node ids are the ordinals
        plain = st.index.compact

        def renumbering():
            n = plain()
            st.index.ids = np.arange(len(st.index.ids), dtype=np.uint64)
            return n
        st.index.compact = renumbering
    refs = [n.ref_doc_id for n in st.nodes]
    dead = set(ids[::3])
    store.delete_documents("ix", sorted(dead))
    kind, alive = st.late_store.calls[-1]
    assert kind == "compact"
    assert alive == [r not in dead for r in refs]                     # the nodes' liveness in ordinal order, before renumbering
    assert len(st.nodes) == sum(alive) and st.n_dead == 0
    assert st.late_store.texts == _texts(st)                          # ordinal o of the store is node o after renumbering
    store.update_documents("ix", [{"doc_id": ids[1], "text": "replaced text of one document", "metadata": {"tag": "a"}}])
    assert st.late_store.texts == _texts(st)


def test_load_rebuilds_the_store_from_every_node_in_ordinal_order(oracle, tmp_path):
    store, _ = _store(oracle)
    ids = store.index_documents("ix", _docs(12, 5))
    store.delete_documents("ix", ids[:3])                              # below the policy: the dead nodes stay
    store.persist("ix", str(tmp_path))
    fresh, rr = _store(oracle)
    fresh.load("ix", str(tmp_path))
    st = fresh.index_map["ix"]
    assert len(st.nodes) == 12 and st.n_dead == 3
    assert st.late_store.texts == _texts(st) and st.late_store.calls[0][1] == 0
    old = st.late_store
    fresh.load("ix", str(tmp_path), overwrite=True)
    assert old.destroyed and fresh.index_map["ix"].late_store is not old
    fresh.delete_index("ix")
    assert rr.stores[-1].destroyed


def test_no_store_without_a_store_capable_reranker(oracle):
    store = vs.VectorStore(HashingEmbedding(64), CompactingOracleEngine(oracle))
    store.index_documents("ix", _docs(5, 1))
    assert store.index_map["ix"].late_store is None


@pytest.mark.parametrize("value,colbert,want", [(None, True, 0), ("", False, 0), ("0", False, 0), ("0.5", True, 500_000_000),
                                                ("8", True, 8_000_000_000)])
def test_store_bytes_from_env(monkeypatch, value, colbert, want):
    if value is None:
        monkeypatch.delenv("KRAG_RERANK_STORE_GB", raising=False)
    else:
        monkeypatch.setenv("KRAG_RERANK_STORE_GB", value)
    assert rerank.store_bytes_from_env(colbert) == want


@pytest.mark.parametrize("value,colbert", [("many", True), ("-1", True), ("nan", True), ("inf", True), ("1", False)])
def test_store_bytes_refusals(monkeypatch, value, colbert):
    monkeypatch.setenv("KRAG_RERANK_STORE_GB", value)
    with pytest.raises(ValueError, match="KRAG_RERANK_STORE_GB"):
        rerank.store_bytes_from_env(colbert)


@pytest.mark.parametrize("value", ["-2", "lots", "4"])
def test_service_exits_on_a_bad_store_budget_before_any_gpu_work(tmp_path, monkeypatch, value):
    """a cross-encoder snapshot: "4" is refused too, since only ColBERT stores passage vectors"""
    import sys
    from kaito_b200 import service
    monkeypatch.setattr(sys, "setswitchinterval", lambda s: None)

    def no_gpu(*a, **k):
        raise AssertionError("the service reached the GPU")
    monkeypatch.setattr(_native, "Context", no_gpu)
    monkeypatch.delenv("KRAG_MODEL_DIR", raising=False)
    monkeypatch.delenv("KRAG_RERANK_PRECISION", raising=False)
    monkeypatch.setenv("EMBEDDING_SOURCE_TYPE", "local")
    monkeypatch.setenv("VECTOR_DB_TYPE", "faiss")
    monkeypatch.setenv("KRAG_RERANK_MODEL_DIR", sts.write(tmp_path, {"config.json": MINILM_CE, "tokenizer_config.json": TOKENIZER_CONFIG}))
    monkeypatch.setenv("KRAG_RERANK_STORE_GB", value)
    with pytest.raises(SystemExit, match=r"reranker '.*' is not supported by this image: KRAG_RERANK_STORE_GB"):
        service.main()


def test_overwrite_load_frees_the_old_store_before_filling_the_new_one(oracle, tmp_path):
    """both stores draw on one budget: the replaced index's store is destroyed before the fresh one is appended to"""
    store, rr = _store(oracle)
    store.index_documents("ix", _docs(8, 6))
    store.persist("ix", str(tmp_path))
    old = store.index_map["ix"].late_store
    events = []
    old.destroy = lambda: events.append("destroy old")
    plain_create = rr.create_store

    def create():
        s = plain_create()
        s.append = lambda texts: (events.append("append fresh"), FakeStore.append(s, texts))
        return s
    rr.create_store = create
    store.load("ix", str(tmp_path), overwrite=True)
    assert events == ["destroy old", "append fresh"]
    assert store.index_map["ix"].late_store.texts == _texts(store.index_map["ix"])


def test_a_store_that_fails_to_compact_is_dropped(oracle, monkeypatch):
    """the engine has compacted: the host renumbers, the store goes, and the index is reranked per call from then on"""
    monkeypatch.setattr(vs, "COMPACT_MIN_DEAD_ROWS", 4)
    monkeypatch.setattr(vs, "COMPACT_DEAD_FRACTION", 0.25)
    store, rr = _store(oracle)
    ids = store.index_documents("ix", _docs(20, 7))
    st = store.index_map["ix"]
    fake = st.late_store

    def broken(alive):
        raise RuntimeError("device error during the moves")
    fake.compact = broken
    store.delete_documents("ix", ids[::2])
    assert st.late_store is None and fake.destroyed
    assert st.n_dead == 0 and all(n.ordinal == i for i, n in enumerate(st.nodes))
    store.retrieve("ix", "retrieval engine", max_node_count=3)
    assert rr.seen[-1] is None                                       # reranked without a store
    store.index_documents("ix", _docs(3, 8))                          # later inserts go on without one
    assert st.late_store is None
