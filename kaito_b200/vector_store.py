"""Host-side mirror of the reference RAGService store classes for the /index and /retrieve
paths, backed by libkaito_rag (CUDA) instead of LlamaIndex + FAISS + bm25s.

Mirrors (paths relative to the reference's presets/ragengine/):
  BaseVectorStore            vector_store/base.py:60-978   (index_documents, retrieve, CRUD, persist/load)
  FaissVectorStoreHandler    vector_store/faiss_store.py:25-50
  HybridRetriever            vector_store/retriever/hybrid_retriever.py:60-237
Same method names, argument meaning and error behaviour (HTTP status + detail strings), so
the reference's own store tests read the same against this class.  The arithmetic of the
path (dense scan, BM25, fusion) runs in the CUDA library through `engine` (a
kaito_b200._native.Context); there is no CPU fallback.
"""
from __future__ import annotations

import hashlib
import json
import os
import threading
import time

import numpy as np

from . import text as _text

FILTER_PUSHDOWN = 0x100   # kaito_rag.h KRAG_FILTER_PUSHDOWN
RAG_MAX_TOP_K = int(os.getenv("RAG_MAX_TOP_K", 300))  # config.py:127
# A delete or update compacts the index (Index.compact: dead rows leave the engine, their text leaves the docstore and the
# snapshots) once the dead rows are at least this share of the rows and at least this many: below that, tombstones cost less
# than moving every live row behind the first dead one.
COMPACT_DEAD_FRACTION = 0.25
COMPACT_MIN_DEAD_ROWS = 65536


class HTTPException(Exception):
    """fastapi.HTTPException stand-in so the store has no web dependency (same fields)."""

    def __init__(self, status_code: int, detail: str):
        super().__init__(f"{status_code}: {detail}")
        self.status_code, self.detail = status_code, detail


def generate_doc_id(text: str) -> str:
    """BaseVectorStore.generate_doc_id, vector_store/base.py:82-85."""
    return hashlib.sha256(text.encode("utf-8")).hexdigest()


def embed_text(text: str, metadata: dict | None) -> str:
    """node.get_content(MetadataMode.EMBED): LlamaIndex's default templates put "key: value" lines,
    a blank line, then the content [3P-unverified]; used for both the embedding and BM25 sides."""
    if not metadata:
        return text
    meta = "\n".join(f"{k}: {v}" for k, v in metadata.items())
    return f"{meta}\n\n{text}"


from .splitter import CodeSplitter, SentenceSplitter   # noqa: E402  (CustomTransformer's two splitters, restated)


class RWLock:
    """Many readers / one writer, writers preferred (aiorwlock.RWLock of the reference, base.py:77-79, with threads
    instead of tasks: FastAPI runs the sync handlers of this service in a thread pool)."""

    def __init__(self):
        self._cv = threading.Condition(threading.Lock())
        self._readers, self._writer, self._waiting_writers = 0, None, 0
        self._depth = 0                      # the writer may re-enter (update -> insert)

    class _Guard:
        def __init__(self, acquire, release):
            self._a, self._r = acquire, release

        def __enter__(self):
            self._a()

        def __exit__(self, *exc):
            self._r()

    def _acquire_read(self):
        me = threading.get_ident()
        with self._cv:
            if self._writer == me:           # the writer reads its own state
                self._depth += 1
                return
            while self._writer is not None or self._waiting_writers:
                self._cv.wait()
            self._readers += 1

    def _release_read(self):
        with self._cv:
            if self._writer == threading.get_ident():
                self._depth -= 1
                return
            self._readers -= 1
            if self._readers == 0:
                self._cv.notify_all()

    def _acquire_write(self):
        me = threading.get_ident()
        with self._cv:
            if self._writer == me:
                self._depth += 1
                return
            self._waiting_writers += 1
            while self._writer is not None or self._readers:
                self._cv.wait()
            self._waiting_writers -= 1
            self._writer, self._depth = me, 1

    def _release_write(self):
        with self._cv:
            self._depth -= 1
            if self._depth == 0:
                self._writer = None
                self._cv.notify_all()

    def reader(self):
        return RWLock._Guard(self._acquire_read, self._release_read)

    def writer(self):
        return RWLock._Guard(self._acquire_write, self._release_write)


class _Node:
    __slots__ = ("node_id", "ref_doc_id", "text", "metadata", "ordinal", "alive", "key")

    def __init__(self, node_id, ref_doc_id, text, metadata, ordinal, key=None):
        self.node_id, self.ref_doc_id, self.text, self.metadata, self.ordinal, self.alive = \
            node_id, ref_doc_id, text, metadata, ordinal, True
        self.key = ordinal if key is None else key   # the engine's node id; stays when a compaction changes the ordinal


class _IndexState:
    def __init__(self, index, late_store=None):
        self.index = index                       # kaito_b200._native.Index (or a test double)
        # the ColBERT reranker's stored passage vectors of this index (kaito_b200.rerank.PassageStore, one entry per ordinal), or
        # None: created by the reranker when KRAG_RERANK_STORE_GB > 0; lives on rank 0 beside the reranker
        self.late_store = late_store
        self.vocab = _text.Vocabulary()
        self.nodes: list[_Node] = []             # by ordinal (== insertion order == engine row)
        self.ref_docs: dict[str, dict] = {}      # doc_id -> {"text", "metadata", "nodes": [ordinal]}
        self.committed = False
        self.next_key = 0                        # engine node id of the next node: len(nodes) until the first compaction
        self.n_dead = 0                          # tombstoned nodes still in `nodes` (and rows in the engine)
        self._filter_cache: dict[str, tuple[int, np.ndarray]] = {}   # filter json -> (nodes covered, allow bitmap)
        self._frag_cache: dict[int, tuple[bytes, bytes]] = {}        # ordinal -> serialised halves of its NodeWithScore
        self._pair_cache: dict[int, tuple] = {}                      # ordinal -> its reranker tokens (encode_passages)

    def pair_passages(self, ordinals, encode) -> list[tuple]:
        """the reranker's tokens of nodes `ordinals` (embed_text of each, as the embedder saw it; `encode` is the reranker's
        encode_passages: a cross-encoder's ids and full length, or a ColBERT model's ids and keep mask): cached per ordinal,
        misses tokenised in one `encode` call.  Two dispatcher threads may fill the cache at once under the store's reader
        lock: nodes are immutable and the tokeniser deterministic, so both compute the same entry, and a dict item assignment
        is atomic under the GIL -- the worst case is a node tokenised twice.  Compaction renumbers ordinals under the writer
        lock and clears the cache there."""
        cache = self._pair_cache
        got = [cache.get(int(o)) for o in ordinals]
        miss = [j for j, g in enumerate(got) if g is None]
        if miss:
            if len(cache) >= 1 << 20:
                cache.clear()
            fresh = encode([embed_text(self.nodes[int(ordinals[j])].text, self.nodes[int(ordinals[j])].metadata) for j in miss])
            for j, f in zip(miss, fresh):
                got[j] = cache[int(ordinals[j])] = f
        return got

    def node_fragments(self, o: int) -> tuple[bytes, bytes]:
        """the JSON of node `o` as a /retrieve result, minus the score: (b'{"doc_id":..,"node_id":..,"text":..,"score":',
        b',"metadata":..,"dense_score":null,"sparse_score":null,"source":null}').  Nodes are immutable once inserted, so the
        halves are cached; a response is then a handful of bytes joins instead of ten dicts through json.dumps."""
        f = self._frag_cache.get(o)
        if f is None:
            n = self.nodes[o]
            dumps = json.dumps
            head = ('{"doc_id":' + dumps(n.ref_doc_id or n.node_id, ensure_ascii=False) + ',"node_id":' + dumps(n.node_id, ensure_ascii=False) +
                    ',"text":' + dumps(n.text, ensure_ascii=False) + ',"score":').encode("utf-8")
            tail = (',"metadata":' + dumps(n.metadata if n.metadata else None, ensure_ascii=False, allow_nan=False, separators=(",", ":")) +
                    ',"dense_score":null,"sparse_score":null,"source":null}').encode("utf-8")
            if len(self._frag_cache) >= 1 << 20:
                self._frag_cache.clear()
            f = self._frag_cache[o] = (head, tail)
        return f

    def allow_bitmap(self, metadata_filter: dict) -> np.ndarray:
        """1 bit per node (ordinal order) whose metadata equals the filter on every key (hybrid_retriever.py:227-235).
        Cached per filter and extended incrementally: a filtered request costs O(new nodes since the last one with the
        same filter), not O(all nodes)."""
        key = json.dumps(metadata_filter, sort_keys=True, default=str)
        n = len(self.nodes)
        done, bm = self._filter_cache.get(key, (0, np.zeros(0, np.uint32)))
        if done < n or bm.size != (n + 31) // 32:
            nb = np.zeros((n + 31) // 32, np.uint32)
            nb[: bm.size] = bm[: nb.size]
            items = list(metadata_filter.items())
            for o in range(done, n):
                md = self.nodes[o].metadata or {}
                if all(md.get(k) == v for k, v in items):
                    nb[o >> 5] |= np.uint32(1 << (o & 31))
            bm = nb
            if len(self._filter_cache) > 256:
                self._filter_cache.clear()
            self._filter_cache[key] = (n, bm)
        return bm


class HybridRetriever:
    """hybrid_retriever.py:60-237: pool size, weights, keyword post-filter, fuse -- on the GPU."""

    def __init__(self, state: _IndexState, embed_model, max_results: int = 10, candidate_multiplier: float = 3.0,
                 vector_weight: float = 0.7, text_weight: float = 0.3, metadata_filter: dict | None = None,
                 filter_pushdown: bool = False, reranker=None, rerank_top_k: int | None = None):
        total = vector_weight + text_weight
        self._vector_weight = vector_weight / total
        self._text_weight = text_weight / total
        self._state, self._embed = state, embed_model
        self._max_results = max_results
        self._candidate_multiplier = max(1.0, candidate_multiplier)
        self._candidate_pool_size = int(max_results * self._candidate_multiplier)
        self._metadata_filter = metadata_filter
        # False (reference): only the keyword list is post-filtered (:227-235).  True: the bitmap restricts the dense and
        # the BM25 scan on the GPU, so every result satisfies the filter (SURVEY.md section 8 f4; not the reference).
        self._filter_pushdown = filter_pushdown
        self.want_components = True          # VectorStore turns this off unless KRAG_COMPONENT_SCORES=1 (saves 10 dicts per query)
        self.last_components: list[dict] = []
        # reranker (kaito_b200.rerank.GpuCrossEncoder, GpuLateInteractionReranker or None): the fused max_results candidates
        # are rescored and the rerank_top_k best kept
        self._reranker, self._rerank_top_k = reranker, rerank_top_k

    def _allow_bitmap(self):
        if not self._metadata_filter:
            return None
        return self._state.allow_bitmap(self._metadata_filter)

    def retrieve(self, query: str) -> list[tuple[_Node, float]]:
        nodes, comps = self.retrieve_batch([query])
        self.last_components = comps[0]
        return nodes[0]

    def retrieve_batch(self, queries: list[str]):
        """`_aretrieve` for a batch of queries that share (index, top_k, filter): ONE embedding forward and ONE engine call.
        Returns (per query: [(node, fused score)], per query: component dicts)."""
        st = self._state
        out = self.retrieve_batch_raw(queries)
        all_nodes, all_comps = [], []
        for b in range(len(queries)):
            c = int(out["count"][b])
            comps = []
            if self.want_components and "dense" in out and "sparse" in out:      # per-result L2^2 / BM25 score as computed by the fuse kernel (NaN = absent)
                for d, s in zip(out["dense"][b, :c], out["sparse"][b, :c]):
                    hd, hs = not np.isnan(d), not np.isnan(s)
                    comps.append({"dense_score": float(d) if hd else None, "sparse_score": float(s) if hs else None,
                                  "source": "both" if hd and hs else ("dense_only" if hd else "sparse_only")})
            all_nodes.append([(st.nodes[int(o)], float(s)) for o, s in zip(out["ordinal"][b, :c], out["final"][b, :c])])
            all_comps.append(comps)
        return all_nodes, all_comps

    def retrieve_batch_raw(self, queries: list[str]) -> dict:
        """the engine's arrays for the batch: "ordinal" [B, k] i64, "final" [B, k] f64, "count" [B] (+ "dense" / "sparse")"""
        st = self._state
        if hasattr(self._embed, "get_query_embedding_batch"):
            q = np.asarray(self._embed.get_query_embedding_batch(queries), np.float32).reshape(len(queries), -1)
        else:
            q = np.stack([np.asarray(self._embed.get_query_embedding(x), np.float32).reshape(-1) for x in queries])
        # BM25 unavailable (empty docstore / nothing committed) -> vector-only fallback (:113-121, :216-218)
        terms = [st.vocab.query_terms(x) for x in queries] if st.committed else None
        allow = self._allow_bitmap() if (terms is not None or self._filter_pushdown) else None
        out = st.index.retrieve(q, terms, self._max_results, cand_mult=self._candidate_multiplier,
                                vector_weight=self._vector_weight, text_weight=self._text_weight,
                                fusion_mode=FILTER_PUSHDOWN if (self._filter_pushdown and allow is not None) else 0,
                                keyword_allow_bitmap=allow)
        if self._reranker is not None:
            out = self._rerank(queries, out)
        return out

    def _rerank(self, queries: list[str], out: dict) -> dict:
        """the engine's arrays cut to the rerank_top_k fused candidates the reranker scores highest, in that order
        (equal scores: fused position ascending); "final" becomes the reranker's score, "dense" / "sparse" follow their
        candidates (they describe the fusion stage)"""
        counts = np.asarray(out["count"])
        cands = [np.asarray(out["ordinal"][b, :int(counts[b])]) for b in range(len(queries))]
        k = self._rerank_top_k
        store = self._state.late_store
        kw = {"store": store} if store is not None else {}
        pos, score = self._reranker.rerank(queries, cands, k, self._state.pair_passages, **kw)
        pos = np.asarray(pos, np.int64)
        valid = pos >= 0
        take = np.where(valid, pos, 0)
        res = {"count": np.minimum(counts, k).astype(counts.dtype),
               "ordinal": np.where(valid, np.take_along_axis(np.asarray(out["ordinal"]), take, 1), -1),
               "final": np.where(valid, np.asarray(score, np.float64), 0.0)}
        for key in ("dense", "sparse"):
            if key in out:
                res[key] = np.where(valid, np.take_along_axis(np.asarray(out[key]), take, 1), np.nan)
        return res


class VectorStore:
    """BaseVectorStore + FaissVectorStoreHandler over the CUDA engine."""

    def __init__(self, embed_model, engine, reranker=None):
        self.embed_model = embed_model
        self.engine = engine
        # optional reranker (KRAG_RERANK_MODEL_DIR: a cross-encoder or ColBERT): /retrieve fuses N = min(max(top_k, KRAG_RERANK_CANDIDATES),
        # RAG_MAX_TOP_K) candidates and returns the top_k the reranker scores highest
        self.reranker = reranker
        self.rerank_candidates = int(os.getenv("KRAG_RERANK_CANDIDATES", "30"))
        self.dimension = embed_model.get_embedding_dimension()   # faiss_store.py:28
        self.index_map: dict[str, _IndexState] = {}
        self.splitter = SentenceSplitter()
        self._code_splitters: dict[str, CodeSplitter] = {}
        self.filter_pushdown = os.getenv("KRAG_FILTER_PUSHDOWN", "0") == "1"
        self.component_scores = os.getenv("KRAG_COMPONENT_SCORES", "0") == "1"
        # many readers / one writer (aiorwlock in the reference, base.py:77-79).  The engine enforces the same
        # discipline per index internally; this lock keeps the host-side docstore (nodes, ref_docs, vocabulary)
        # consistent with the engine rows for the whole of a retrieve / chat / persist, as the reference's reader
        # lock does (base.py:917-919)
        self._rw = RWLock()

    # ------------------------------------------------------------------ /index
    def index_documents(self, index_name: str, documents: list[dict]) -> list[str]:
        """base.py:90-97: create on first use, else append with per-document dedupe (:99-131)."""
        with self._rw.writer():
            st = self.index_map.get(index_name)
            if st is None:
                st = _IndexState(self.engine.create_index(index_name, self.dimension), self._new_late_store())
                self.index_map[index_name] = st
            ids, fresh, fresh_ids = [], [], set()
            for doc in documents:
                doc_id = generate_doc_id(doc["text"])
                ids.append(doc_id)
                if doc_id in st.ref_docs or doc_id in fresh_ids:
                    continue                                   # "already exists ... Skipping." (:123-126)
                fresh_ids.add(doc_id)
                fresh.append((doc_id, doc["text"], doc.get("metadata") or {}))
            if fresh:
                self._insert(st, fresh)
            return ids

    def _new_late_store(self):
        """the reranker's passage vector store for a new index, or None (no ColBERT reranker, or storing off)"""
        create = getattr(self.reranker, "create_store", None)
        return create() if create is not None else None

    @staticmethod
    def _drop_store(st: _IndexState):
        store, st.late_store = st.late_store, None
        if store is not None:
            store.destroy()

    @staticmethod
    def _drop_state(st: _IndexState):
        st.index.drop()
        VectorStore._drop_store(st)

    def _insert(self, st: _IndexState, docs, replace: bool = False):
        """Chunk, analyse, embed and append `docs`; the host docstore is published only after the embedder and the
        engine accepted the whole batch, so a failure (remote embedder error, 501 for code splitting, engine error)
        leaves neither a listed-but-unretrievable document nor ordinals that a later insert would reuse."""
        for _, _, metadata in docs:                                     # validate the whole batch before any work
            if metadata.get("split_type") == "code" and not metadata.get("language"):
                raise ValueError("Language not specified in node metadata.")      # custom_transformer.py:39-41
        node_ids, texts, offs, tids, tfs, dls, new_nodes, new_refs = [], [], [0], [], [], [], [], {}
        base = len(st.nodes)
        for doc_id, text, metadata in docs:
            ords = []
            for i, chunk in enumerate(self.split_document(text, metadata)):
                ordinal = base + len(new_nodes)
                key = st.next_key + len(new_nodes)
                new_nodes.append(_Node(f"{doc_id}-{i}", doc_id, chunk, metadata, ordinal, key))
                et = embed_text(chunk, metadata)
                texts.append(et)
                t_ids, t_tf, dl = st.vocab.doc_terms(et)     # may grow the vocabulary: unused ids are harmless
                tids.append(t_ids); tfs.append(t_tf); dls.append(dl)
                offs.append(offs[-1] + len(t_ids))
                node_ids.append(key)
                ords.append(ordinal)
            new_refs[doc_id] = {"text": text, "metadata": metadata, "nodes": ords}
        vecs = np.asarray(self.embed_model.get_text_embedding_batch(texts), np.float32)
        store = st.late_store
        try:
            if store is not None:               # ordinals base .. : the texts rerank() would encode for them
                store.append(texts)
            st.index.add(np.asarray(node_ids, np.uint64), vecs, np.asarray(offs, np.int64),
                         np.concatenate(tids) if tids else np.zeros(0, np.uint32),
                         np.concatenate(tfs) if tfs else np.zeros(0, np.uint16), np.asarray(dls, np.uint32))
        except BaseException:
            if store is not None:
                store.truncate(base)
            raise
        # the rows are in the engine: publish.  (A failing commit below leaves the index "uncommitted": /retrieve takes
        # the reference's vector-only fallback until the next successful commit.)
        st.nodes.extend(new_nodes)
        st.next_key += len(new_nodes)
        old = {d: st.ref_docs.get(d) for d in new_refs} if replace else {}
        st.ref_docs.update(new_refs)
        st.committed = False
        self._commit(st)
        return old

    def split_document(self, text: str, metadata: dict) -> list[str]:
        """CustomTransformer.split_node (custom_transformer.py:34-49): CodeSplitter(language) for split_type == "code" (one
        splitter per language, cached), SentenceSplitter() otherwise -- with the metadata-aware chunk budget LlamaIndex applies
        (the "key: value" block prepended for the embedder counts against chunk_size)."""
        if metadata.get("split_type", "default") == "code":
            lang = metadata.get("language", "")
            if not lang:
                raise ValueError("Language not specified in node metadata.")
            sp = self._code_splitters.get(lang)
            if sp is None:
                sp = self._code_splitters[lang] = CodeSplitter(language=lang)
            return sp.split(text) or [text]
        meta_str = "\n".join(f"{k}: {v}" for k, v in metadata.items()) if metadata else ""
        return self.splitter.split(text, meta_str) or [text]

    def _commit(self, st: _IndexState):
        # the reference rebuilds BM25 on every query (hybrid_retriever.py:104-130); here once per mutation
        st.index.commit(max(1, len(st.vocab)))
        st.committed = True

    def _maybe_compact(self, st: _IndexState):
        """after a committed delete / update (writer lock held): compact the engine index when enough of it is dead, then
        drop the dead nodes from the host mirror and renumber the live ones as the engine did (order kept)"""
        if (st.n_dead < COMPACT_MIN_DEAD_ROWS or st.n_dead < COMPACT_DEAD_FRACTION * len(st.nodes)
                or not hasattr(st.index, "compact")):      # an engine without compaction keeps its tombstones
            return
        st.index.compact()
        if st.late_store is not None:           # the same renumbering as below: live ordinals in order
            try:
                st.late_store.compact([n.alive for n in st.nodes])
            except Exception:
                # the engine has compacted, so the host renumbers below whatever happens here; a store that could not
                # follow (a device error, possibly part way through its moves) no longer matches the ordinals: drop it,
                # and the index is reranked per call, with the same scores
                self._drop_store(st)
        live = [n for n in st.nodes if n.alive]
        # the sharded engine's node ids are the ordinals: its compaction renumbers them too, and the next node gets n_live
        renumber = getattr(st.index, "compact_renumbers_keys", False)
        remap = {}
        for i, n in enumerate(live):
            remap[n.ordinal] = i
            n.ordinal = i
            if renumber:
                n.key = i
        if renumber:
            st.next_key = len(live)
        st.nodes = live
        for rec in st.ref_docs.values():
            rec["nodes"] = [remap[o] for o in rec["nodes"]]
        st.n_dead = 0
        st._frag_cache.clear()           # these caches are keyed by ordinal
        st._pair_cache.clear()
        st._filter_cache.clear()

    # --------------------------------------------------------------- /retrieve
    def _retriever(self, st: _IndexState, top_k: int, metadata_filter: dict | None) -> HybridRetriever:
        """the retriever every /retrieve path uses: top_k fused results, or with a reranker N fused candidates cut to top_k"""
        if self.reranker is None:
            return HybridRetriever(st, self.embed_model, max_results=top_k, metadata_filter=metadata_filter,
                                   filter_pushdown=self.filter_pushdown)
        n = min(max(top_k, self.rerank_candidates), RAG_MAX_TOP_K)
        return HybridRetriever(st, self.embed_model, max_results=n, metadata_filter=metadata_filter,
                               filter_pushdown=self.filter_pushdown, reranker=self.reranker, rerank_top_k=top_k)

    def retrieve(self, index_name: str, query: str, max_node_count: int = 5, metadata_filter: dict | None = None):
        """base.py:870-978."""
        if index_name not in self.index_map:
            raise HTTPException(404, f"No such index: '{index_name}' exists.")
        try:
            if not query or query.strip() == "":
                raise HTTPException(400, "Query string cannot be empty.")
            top_k = min(max_node_count, RAG_MAX_TOP_K)
            st = self.index_map[index_name]
            retriever = self._retriever(st, top_k, metadata_filter)
            t0 = time.time()
            with self._rw.reader():         # base.py:917-919: reader lock around the retrieval
                nodes = retriever.retrieve(query)
                results = [{"doc_id": n.ref_doc_id or n.node_id, "node_id": n.node_id, "text": n.text, "score": s,
                            "metadata": n.metadata if n.metadata else None} for n, s in nodes]
            self.last_retrieve_seconds = time.time() - t0
            if self.component_scores:       # KRAG_COMPONENT_SCORES=1: fill the optional fields of models.NodeWithScore
                for r, extra in zip(results, retriever.last_components):
                    r.update(extra)
            return {"query": query, "results": results, "count": len(results)}
        except HTTPException:
            raise
        except Exception as e:  # same envelope as base.py:972-978
            raise HTTPException(500, f"Retrieve failed: {e}")

    def retrieve_batch(self, index_name: str, queries: list[str], max_node_count: int = 5, metadata_filter: dict | None = None):
        """retrieve() for several queries against the same index with the same top_k and filter, answered by one engine call
        (kaito_b200.batcher coalesces concurrent /retrieve requests into this).  Returns one response dict per query; a
        blank query yields the reference's 400 for that entry only."""
        if index_name not in self.index_map:
            raise HTTPException(404, f"No such index: '{index_name}' exists.")
        bad = HTTPException(400, "Query string cannot be empty.")
        live = [i for i, q in enumerate(queries) if q and q.strip() != ""]
        outs: list = [bad] * len(queries)
        if not live:
            return outs
        try:
            top_k = min(max_node_count, RAG_MAX_TOP_K)
            t0 = time.time()
            with self._rw.reader():
                st = self.index_map[index_name]
                retriever = self._retriever(st, top_k, metadata_filter)
                retriever.want_components = self.component_scores
                nodes, comps = retriever.retrieve_batch([queries[i] for i in live])
                for j, i in enumerate(live):
                    results = [{"doc_id": n.ref_doc_id or n.node_id, "node_id": n.node_id, "text": n.text, "score": s,
                                "metadata": n.metadata if n.metadata else None} for n, s in nodes[j]]
                    if self.component_scores and comps[j]:
                        for r, extra in zip(results, comps[j]):
                            r.update(extra)
                    outs[i] = {"query": queries[i], "results": results, "count": len(results)}
            self.last_retrieve_seconds = (time.time() - t0) / len(live)
            return outs
        except HTTPException:
            raise
        except Exception as e:
            raise HTTPException(500, f"Retrieve failed: {e}")

    def retrieve_batch_bytes(self, index_name: str, queries: list[str], max_node_count: int = 5, metadata_filter: dict | None = None):
        """retrieve_batch() with the responses already serialised: per query (json bytes, count, fused scores) or the
        HTTPException of that entry.  The bytes parse to exactly what retrieve_batch() returns plus the null defaults of
        models.NodeWithScore; they are assembled from cached per-node fragments (the HTTP fast path and the front-end workers
        forward them untouched)."""
        if self.component_scores:                       # optional per-result fields: take the dict path
            outs = self.retrieve_batch(index_name, queries, max_node_count, metadata_filter)
            res = []
            for o in outs:
                if isinstance(o, Exception):
                    res.append(o); continue
                for r in o["results"]:
                    r.setdefault("dense_score", None); r.setdefault("sparse_score", None); r.setdefault("source", None)
                res.append((json.dumps(o, ensure_ascii=False, allow_nan=False, separators=(",", ":")).encode("utf-8"), o["count"],
                            [r["score"] for r in o["results"]]))
            return res
        if index_name not in self.index_map:
            raise HTTPException(404, f"No such index: '{index_name}' exists.")
        bad = HTTPException(400, "Query string cannot be empty.")
        live = [i for i, q in enumerate(queries) if q and q.strip() != ""]
        outs: list = [bad] * len(queries)
        if not live:
            return outs
        try:
            top_k = min(max_node_count, RAG_MAX_TOP_K)
            t0 = time.time()
            with self._rw.reader():
                st = self.index_map[index_name]
                retriever = self._retriever(st, top_k, metadata_filter)
                out = retriever.retrieve_batch_raw([queries[i] for i in live])
                counts, ords, finals = out["count"].tolist(), out["ordinal"].tolist(), out["final"].tolist()
                frag = st.node_fragments
                for j, i in enumerate(live):
                    c = counts[j]
                    scores = finals[j][:c]
                    parts = []
                    for o, sc in zip(ords[j][:c], scores):
                        if sc != sc or sc in (float("inf"), float("-inf")):
                            raise ValueError("Out of range float values are not JSON compliant")
                        head, tail = frag(o)
                        parts.append(head + repr(sc).encode("ascii") + tail)
                    body = b'{"query":' + json.dumps(queries[i], ensure_ascii=False).encode("utf-8") + b',"results":[' + b",".join(parts) + \
                           b'],"count":' + str(c).encode("ascii") + b"}"
                    outs[i] = (body, c, scores)
            self.last_retrieve_seconds = (time.time() - t0) / len(live)
            return outs
        except HTTPException:
            raise
        except Exception as e:
            raise HTTPException(500, f"Retrieve failed: {e}")

    # ------------------------------------------------- /v1/chat/completions
    def dense_candidates(self, index_name: str, query: str, top_k: int) -> list[tuple[_Node, float]]:
        """index.as_retriever(similarity_top_k=top_k) of the chat engine (base.py:376-391): exact dense kNN, faiss
        scores = squared L2 distances, ascending."""
        q = np.asarray(self.embed_model.get_query_embedding(query), np.float32).reshape(1, -1)
        with self._rw.reader():
            st = self.index_map[index_name]
            k = max(1, min(top_k, sum(1 for n in st.nodes if n.alive)))
            dist, ordn = st.index.search_dense(q, k)
            return [(st.nodes[int(o)], float(d)) for d, o in zip(dist[0], ordn[0]) if o >= 0]

    def chat_completion(self, request: dict, llm, cfg: dict | None = None) -> dict:
        """base.py:180-477 -- see kaito_b200/chat.py"""
        from . import chat
        return chat.chat_completion(self, llm, request, cfg)

    # ------------------------------------------------------------------- CRUD
    def list_indexes(self) -> list[str]:
        return list(self.index_map.keys())

    def document_exists(self, index_name: str, doc_id: str) -> bool:
        st = self.index_map.get(index_name)
        return bool(st and doc_id in st.ref_docs)

    def list_documents_in_index(self, index_name: str, limit: int = 10, offset: int = 0, max_text_length: int | None = 1000,
                                metadata_filter: dict | None = None):
        if index_name not in self.index_map:
            raise HTTPException(404, f"No such index: '{index_name}' exists.")
        st = self.index_map[index_name]
        docs = []
        for doc_id, d in st.ref_docs.items():
            if metadata_filter and not all(d["metadata"].get(k) == v for k, v in metadata_filter.items()):
                continue
            docs.append((doc_id, d))
        total = len(docs)
        out = []
        for doc_id, d in docs[offset:offset + limit]:
            t = d["text"]
            trunc = max_text_length is not None and len(t) > max_text_length
            out.append({"doc_id": doc_id, "text": t[:max_text_length] if trunc else t, "metadata": d["metadata"],
                        "hash_value": generate_doc_id(t), "is_truncated": trunc})
        return {"documents": out, "count": len(out), "total_items": total}

    def delete_documents(self, index_name: str, doc_ids: list[str]):
        if index_name not in self.index_map:
            raise HTTPException(404, f"No such index: '{index_name}' exists.")
        with self._rw.writer():
            st = self.index_map[index_name]
            deleted, missing, rows = [], [], []
            for d in doc_ids:
                rec = st.ref_docs.pop(d, None)
                if rec is None:
                    missing.append(d)
                    continue
                deleted.append(d)
                for o in rec["nodes"]:
                    st.nodes[o].alive = False
                    rows.append(st.nodes[o].key)
            if rows:
                st.index.remove(np.asarray(rows, np.uint64))
                st.n_dead += len(rows)
                self._commit(st)
                self._maybe_compact(st)
            return {"deleted_doc_ids": deleted, "not_found_doc_ids": missing}

    def update_documents(self, index_name: str, documents: list[dict]):
        """base.py:529-561 semantics: by doc_id; unchanged text -> unchanged, else delete + re-insert."""
        if index_name not in self.index_map:
            raise HTTPException(404, f"No such index: '{index_name}' exists.")
        with self._rw.writer():
            st = self.index_map[index_name]
            updated, unchanged, missing = [], [], []
            for doc in documents:
                rec = st.ref_docs.get(doc.get("doc_id", ""))
                if rec is None:
                    missing.append(doc)
                elif rec["text"] == doc["text"] and (doc.get("metadata") or {}) == rec["metadata"]:
                    unchanged.append(doc)
                else:
                    # new rows first, old rows tombstoned only once the replacement is in: a failing embed/add leaves
                    # the document as it was (the reference deletes first, base.py:529-561, and can lose it)
                    old_rows = list(rec["nodes"])
                    self._insert(st, [(doc["doc_id"], doc["text"], doc.get("metadata") or {})], replace=True)
                    for o in old_rows:
                        st.nodes[o].alive = False
                    st.index.remove(np.asarray([st.nodes[o].key for o in old_rows], np.uint64))
                    st.n_dead += len(old_rows)
                    self._commit(st)
                    updated.append(doc)
            if updated:
                self._maybe_compact(st)
            return {"updated_documents": updated, "unchanged_documents": unchanged, "not_found_documents": missing}

    def delete_index(self, index_name: str):
        if index_name not in self.index_map:
            raise HTTPException(404, f"No such index: '{index_name}' exists.")
        with self._rw.writer():
            self._drop_state(self.index_map.pop(index_name))

    # -------------------------------------------------------- persist / load
    def persist(self, index_name: str, path: str):
        """base.py:779-809. Own format: the engine snapshot + docstore.json (SURVEY.md section 5)."""
        if index_name not in self.index_map:
            raise HTTPException(404, f"No such index: '{index_name}' exists.")
        with self._rw.reader():             # engine snapshot and docstore.json describe the same state
            st = self.index_map[index_name]
            os.makedirs(path, exist_ok=True)
            st.index.persist(path)
            ds = {"version": 1, "vocab": st.vocab.terms, "ref_docs": st.ref_docs,
                  "nodes": [[n.node_id, n.ref_doc_id, n.text, n.metadata, n.alive] for n in st.nodes]}
            if any(n.key != n.ordinal for n in st.nodes):    # engine node ids; absent: key = ordinal (every earlier snapshot)
                ds["keys"] = [n.key for n in st.nodes]
            with open(os.path.join(path, "docstore.json"), "w") as f:
                json.dump(ds, f)

    def load(self, index_name: str, path: str, overwrite: bool = False):
        """base.py:811-868."""
        if index_name in self.index_map and not overwrite:
            raise HTTPException(409, f"Index '{index_name}' already exists. Use a different name or delete the existing index first.")
        if not os.path.exists(path):        # base.py:841-845
            raise HTTPException(404, f"Path does not exist: {path}")
        try:
            with open(os.path.join(path, "docstore.json")) as f:
                ds = json.load(f)
            with self._rw.writer():
                # load beside the live index (under a scratch engine name) and swap only on success: a corrupt snapshot
                # must not destroy what is being served (the reference replaces index_map[name] after the load, :847-860)
                fresh = _IndexState(self.engine.load_index(index_name, path))
                try:
                    for t in ds["vocab"]:
                        fresh.vocab.add(t)
                    fresh.ref_docs = ds["ref_docs"]
                    keys = ds.get("keys")
                    for i, (nid, rid, text, meta, alive) in enumerate(ds["nodes"]):
                        n = _Node(nid, rid, text, meta, i, keys[i] if keys else i)
                        n.alive = alive
                        fresh.nodes.append(n)
                    fresh.next_key = max(keys) + 1 if keys else len(fresh.nodes)
                    fresh.n_dead = sum(1 for n in fresh.nodes if not n.alive)
                    fresh.committed = True
                    # the snapshot holds no passage vectors: every node, dead ones too (compaction drops them), in ordinal order.
                    # The index being replaced gives its stored vectors back to the shared budget first (it keeps serving,
                    # reranked per call, should this load still fail), so the fresh store can take their room.
                    if index_name in self.index_map:
                        self._drop_store(self.index_map[index_name])
                    fresh.late_store = self._new_late_store()
                    if fresh.late_store is not None:
                        fresh.late_store.append([embed_text(n.text, n.metadata) for n in fresh.nodes])
                except Exception:
                    self._drop_state(fresh)
                    raise
                old = self.index_map.get(index_name)
                self.index_map[index_name] = fresh
                if old is not None:
                    self._drop_state(old)
        except HTTPException:
            raise
        except Exception as e:
            raise HTTPException(500, f"Loading failed: {e}")
