"""RAGService HTTP surface over the CUDA engine -- the drop-in for presets/ragengine/main.py that the
unmodified KAITO ragengine controller deploys (pod contract: SURVEY.md section 8 b1, INTEGRATION.md).

Routes, status codes and detail strings follow the reference (presets/ragengine/main.py): GET /metrics :165,
GET /health :180, POST /index :217, POST /v1/chat/completions :275, GET /indexes :356,
GET /indexes/{name}/documents :393, POST /indexes/{name}/documents :495,
POST /indexes/{name}/documents/delete :546, POST /persist/{name} :596, POST /load/{name} :652,
POST /retrieve :704, DELETE /indexes/{name} :774.  Unknown JSON fields are ignored (test/rage2e sends
`context_token_ratio`, rag_test.go:1254).  Prometheus metric names: metrics/prometheus_metrics.py:27-201.

The host language north_star asks for is Go; no Go toolchain exists in this image, so the host is Python
like the reference service itself, and binds the same C ABI a cgo host would (INTEGRATION.md).
"""
from __future__ import annotations

import json
import os
import time
from urllib.parse import unquote

from fastapi import FastAPI, HTTPException, Query, Request, Response
from fastapi.responses import JSONResponse as _JSON
from prometheus_client import CONTENT_TYPE_LATEST, CollectorRegistry, Counter, Gauge, Histogram, generate_latest
from pydantic import BaseModel, Field

from . import vector_store as vs

RAG_MAX_TOP_K = vs.RAG_MAX_TOP_K


# --------------------------------------------------------------------------- wire models (models.py:24-93)
class Document(BaseModel):
    doc_id: str = Field(default="")
    text: str
    metadata: dict | None = Field(default_factory=dict)
    hash_value: str | None = None
    is_truncated: bool = False


class IndexRequest(BaseModel):
    index_name: str
    documents: list[Document]


class UpdateDocumentRequest(BaseModel):
    documents: list[Document]


class DeleteDocumentRequest(BaseModel):
    doc_ids: list[str]


class RetrieveRequest(BaseModel):
    index_name: str
    query: str
    max_node_count: int = Field(default=5, ge=1, le=RAG_MAX_TOP_K)
    metadata_filter: dict | None = None


class NodeWithScore(BaseModel):          # models.py:63-71; the reference's retrieve leaves the three optional scores unset
    doc_id: str
    node_id: str
    text: str
    score: float
    dense_score: float | None = None
    sparse_score: float | None = None
    source: str | None = None            # "both", "dense_only", "sparse_only"
    metadata: dict | None = None


class RetrieveResponse(BaseModel):
    query: str
    results: list[NodeWithScore]
    count: int


class ListDocumentsResponse(BaseModel):
    documents: list[Document]
    count: int
    total_items: int


class UpdateDocumentResponse(BaseModel):
    updated_documents: list[Document]
    unchanged_documents: list[Document]
    not_found_documents: list[Document]


class DeleteDocumentResponse(BaseModel):
    deleted_doc_ids: list[str]
    not_found_doc_ids: list[str]


class HealthStatus(BaseModel):
    status: str
    detail: str | None = None


def env_config() -> dict:
    """config.py names, plus the spellings the controller actually injects (SURVEY.md section 0 Q8:
    manifests.go:171-194 sets MODEL_ID / EMBEDDING_TYPE, the reference service reads
    LOCAL_EMBEDDING_MODEL_ID / EMBEDDING_SOURCE_TYPE -- both are honoured here)."""
    g = os.getenv
    return {
        "embedding_source": g("EMBEDDING_SOURCE_TYPE") or g("EMBEDDING_TYPE") or "local",
        "embedding_model": g("LOCAL_EMBEDDING_MODEL_ID") or g("MODEL_ID") or "BAAI/bge-small-en-v1.5",
        "remote_embedding_url": g("REMOTE_EMBEDDING_URL", "http://localhost:5000/embedding"),
        "remote_embedding_access_secret": g("REMOTE_EMBEDDING_ACCESS_SECRET", "default-access-secret"),
        "vector_db_type": g("VECTOR_DB_TYPE", "faiss"),
        "persist_dir": g("DEFAULT_VECTOR_DB_PERSIST_DIR", "storage"),
        "llm_inference_url": g("LLM_INFERENCE_URL"),
        "device_id": int(g("KRAG_DEVICE_ID", "0")),
    }


# --------------------------------------------------------------- Prometheus metrics (metrics/prometheus_metrics.py:27-330)
# Every metric the reference registers -- name, kind, labels, buckets -- including the rag_hybrid_* family it defines for its
# dashboards but never observes (kept registered so that scrapes and dashboards see the same series set).
_B_DEFAULT = None
_B_SCORE = (0.1, 0.2, 0.3, 0.35, 0.4, 0.45, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0)
_B_HSCORE = (0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 0.95, 1.0)
_B_CAND = (0, 1, 2, 3, 5, 10, 20, 50, 100)
_B_CNT = (0, 1, 2, 3, 5, 10, 20, 50)
METRIC_SPEC = [
    ("rag_embedding_latency_seconds", "H", ("status", "mode"), _B_DEFAULT, "Time to embed in seconds"),
    ("rag_embedding_requests", "C", ("status", "mode"), None, "Count of successful/failed embed requests"),
    ("rag_chat_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call '/v1/chat/completions' API in seconds"),
    ("rag_chat_requests", "C", ("status",), None, "Count of successful/failed calling '/v1/chat/completions' requests"),
    ("rag_index_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call '/index' API in seconds"),
    ("rag_index_requests", "C", ("status",), None, "Count of successful/failed calling '/index' requests"),
    ("rag_indexes_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call '/indexes' API in seconds"),
    ("rag_indexes_requests", "C", ("status",), None, "Count of successful/failed calling '/indexes' requests"),
    ("rag_indexes_document_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call get '/indexes/{index_name}/documents' API in seconds"),
    ("rag_indexes_document_requests", "C", ("status",), None, "Count of successful/failed calling get '/indexes/{index_name}/documents' requests"),
    ("rag_indexes_update_document_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call post '/indexes/{index_name}/documents' API in seconds"),
    ("rag_indexes_update_document_requests", "C", ("status",), None, "Count of successful/failed calling post '/indexes/{index_name}/documents' requests"),
    ("rag_indexes_retrieve_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call post '/retrieve' API in seconds"),
    ("rag_indexes_retrieve_requests", "C", ("status",), None, "Count of successful/failed calling post '/retrieve' requests"),
    ("rag_indexes_delete_document_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call '/indexes/{index_name}/documents/delete' API in seconds"),
    ("rag_indexes_delete_document_requests", "C", ("status",), None, "Count of successful/failed calling '/indexes/{index_name}/documents/delete' requests"),
    ("rag_persist_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call '/persist/{index_name}' API in seconds"),
    ("rag_persist_requests", "C", ("status",), None, "Count of successful/failed calling '/persist/{index_name}' requests"),
    ("rag_load_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call '/load/{index_name}' API in seconds"),
    ("rag_load_requests", "C", ("status",), None, "Count of successful/failed calling '/load/{index_name}' requests"),
    ("rag_delete_index_latency_seconds", "H", ("status",), _B_DEFAULT, "Time to call delete '/indexes/{index_name}' API in seconds"),
    ("rag_delete_index_requests", "C", ("status",), None, "Count of successful/failed calling delete '/indexes/{index_name}' requests"),
    ("e2e_request", "C", ("status",), None, "Total number of all processed requests"),
    ("e2e_request_latency_seconds", "H", ("status",), _B_DEFAULT, "End to end request latency in seconds"),
    ("num_requests_running", "G", (), None, "Number of requests currently being processed"),
    ("rag_vector_store_operation_latency_seconds", "H", ("operation", "status"), (0.005, 0.01, 0.025, 0.05, 0.1, 0.25, 0.5, 1.0, 2.5, 5.0, 10.0),
     "Latency of vector store backend operations (insert, query, delete)"),
    ("rag_retrieve_result_count", "H", (), (0, 1, 2, 3, 5, 10, 20, 50, 100, 200, 300), "Number of document chunks returned per retrieve call"),
    ("rag_lowest_source_score", "H", (), _B_SCORE, "Score of the lowest scoring source node (typically the most relevant)"),
    ("rag_avg_source_score", "H", (), _B_SCORE, "Average score of all retrieved source documents in RAG queries"),
    ("rag_hybrid_search_mode", "C", ("search_mode",), None, "Number of retrieve calls by search mode"),
    ("rag_hybrid_retrieve_latency_seconds", "H", (), (0.005, 0.01, 0.025, 0.05, 0.1, 0.25, 0.5, 1.0, 2.5, 5.0),
     "End-to-end latency of hybrid retrieve (dense+sparse encode, query, fusion)"),
    ("rag_hybrid_retrieve_latency_avg_seconds", "G", (), None, "Running average latency of hybrid retrieve calls (sum / count)"),
    ("rag_hybrid_top_score", "H", (), _B_HSCORE, "Highest (best) fused score among results per hybrid retrieve call"),
    ("rag_hybrid_median_score", "H", (), _B_HSCORE, "Median fused score of results per hybrid retrieve call"),
    ("rag_hybrid_score_spread", "H", (), (0.0, 0.05, 0.1, 0.15, 0.2, 0.3, 0.4, 0.5, 0.7, 1.0), "Score spread (max - min) per hybrid retrieve call"),
    ("rag_hybrid_top_k_requested", "H", (), (1, 2, 3, 5, 10, 20, 50, 100), "The top_k value requested per hybrid retrieve call"),
    ("rag_hybrid_sparse_top_k", "H", (), (3, 6, 9, 15, 30, 60, 150, 300), "The sparse_top_k (prefetch) value used per hybrid retrieve call"),
    ("rag_hybrid_dense_candidates", "H", (), _B_CAND, "Number of dense (vector) candidate nodes returned before fusion"),
    ("rag_hybrid_sparse_candidates", "H", (), _B_CAND, "Number of sparse (BM25) candidate nodes returned before fusion"),
    ("rag_hybrid_overlap_count", "H", (), _B_CNT, "Number of final result nodes that appear in BOTH dense and sparse results"),
    ("rag_hybrid_dense_only_count", "H", (), _B_CNT, "Number of final result nodes that came from dense (vector) search only"),
    ("rag_hybrid_sparse_only_count", "H", (), _B_CNT, "Number of final result nodes that came from sparse (BM25) search only"),
]


def build_metrics(reg: CollectorRegistry) -> dict:
    out = {}
    for name, kind, labels, buckets, doc in METRIC_SPEC:
        if kind == "H":
            kw = {} if buckets is None else {"buckets": buckets}
            out[name] = Histogram(name, doc, labelnames=list(labels), registry=reg, **kw)
        elif kind == "C":
            out[name] = Counter(name, doc, labelnames=list(labels), registry=reg)
        else:
            out[name] = Gauge(name, doc, registry=reg)
    return out


def create_app(store: vs.VectorStore, cfg: dict | None = None, llm=None) -> FastAPI:
    cfg = cfg or env_config()
    from . import chat as _chat
    chat_cfg = {**_chat.chat_config(), **{k: v for k, v in cfg.items() if k in _chat.chat_config()}}
    if llm is None and chat_cfg.get("llm_inference_url"):
        llm = _chat.LLMClient(chat_cfg["llm_inference_url"], chat_cfg["llm_access_secret"], chat_cfg["llm_context_window"])
    app = FastAPI(title="KAITO RAGEngine service (H100-native)")
    reg = CollectorRegistry()
    mx = build_metrics(reg)
    M = {"index": ("rag_index_latency_seconds", "rag_index_requests"), "indexes": ("rag_indexes_latency_seconds", "rag_indexes_requests"),
         "documents": ("rag_indexes_document_latency_seconds", "rag_indexes_document_requests"),
         "update": ("rag_indexes_update_document_latency_seconds", "rag_indexes_update_document_requests"),
         "retrieve": ("rag_indexes_retrieve_latency_seconds", "rag_indexes_retrieve_requests"),
         "delete_doc": ("rag_indexes_delete_document_latency_seconds", "rag_indexes_delete_document_requests"),
         "persist": ("rag_persist_latency_seconds", "rag_persist_requests"), "load": ("rag_load_latency_seconds", "rag_load_requests"),
         "delete": ("rag_delete_index_latency_seconds", "rag_delete_index_requests"), "chat": ("rag_chat_latency_seconds", "rag_chat_requests")}
    M = {k: (mx[h], mx[c]) for k, (h, c) in M.items()}
    e2e_total, e2e_lat, running = mx["e2e_request"], mx["e2e_request_latency_seconds"], mx["num_requests_running"]
    vs_lat, res_count = mx["rag_vector_store_operation_latency_seconds"], mx["rag_retrieve_result_count"]
    low_score, avg_score = mx["rag_lowest_source_score"], mx["rag_avg_source_score"]
    emb_lat, emb_cnt = mx["rag_embedding_latency_seconds"], mx["rag_embedding_requests"]
    emb_mode = "remote" if str(cfg.get("embedding_source", "local")).lower() == "remote" else "local"   # MODE_LOCAL / MODE_REMOTE
    app.state.store, app.state.registry = store, reg
    # request coalescer (kaito_b200/batcher.py): concurrent /retrieve calls -> one engine call per (index, top_k, filter) group
    from .batcher import RetrieveBatcher
    batcher = RetrieveBatcher(store) if hasattr(store, "retrieve_batch") else None
    app.state.batcher = batcher

    TRACKED = ("/index", "/indexes", "/persist", "/load", "/retrieve", "/v1/chat/completions")

    class TrackRequests:
        """main.py:97-128 (in-flight gauge + end-to-end latency on the tracked paths; status = the handler returned) as a plain
        ASGI middleware: Starlette's BaseHTTPMiddleware costs an anyio task group and two memory streams per request, which at
        thousands of requests per second is most of the event loop's time"""

        def __init__(self, inner):
            self.inner = inner

        async def __call__(self, scope, receive, send):
            if scope["type"] != "http" or not any(scope["path"].startswith(p) for p in TRACKED):
                return await self.inner(scope, receive, send)
            running.inc()
            t0 = time.perf_counter()
            status = "failure"
            try:
                await self.inner(scope, receive, send)
                status = "success"
            finally:
                running.dec()
                e2e_lat.labels(status).observe(time.perf_counter() - t0)
                e2e_total.labels(status).inc()

    def _observe_retrieve(status, seconds, out):
        h, c = M["retrieve"]
        c.labels(status).inc(); h.labels(status).observe(seconds)
        if out is not None:
            res_count.observe(out["count"])
            vs_lat.labels("query", "success").observe(getattr(store, "last_retrieve_seconds", 0.0))
            scores = [r["score"] for r in out["results"]]
            if scores:
                low_score.observe(min(scores)); avg_score.observe(sum(scores) / len(scores))

    app.state.observe_retrieve = _observe_retrieve        # the front-end workers' RPC server books its requests here (rpc.py)
    if batcher is not None and batcher.enabled and os.getenv("KRAG_FAST_RETRIEVE", "1") != "0":
        # well-formed POST /retrieve requests are answered below FastAPI's routing stack (kaito_b200/fast_retrieve.py); anything
        # else -- including every request FastAPI would reject -- still reaches the route below
        from .fast_retrieve import FastRetrieve
        app.add_middleware(FastRetrieve, submit=batcher.submit_bytes if hasattr(store, "retrieve_batch_bytes") else batcher.submit,
                           observe=_observe_retrieve, max_top_k=RAG_MAX_TOP_K,
                           http_exception_types=(vs.HTTPException, HTTPException))
    app.add_middleware(TrackRequests)

    def run(kind, fn):
        """observe latency/status like the reference's per-route try/finally blocks"""
        h, c = M[kind]
        t0 = time.perf_counter()
        try:
            out = fn()
            c.labels("success").inc(); h.labels("success").observe(time.perf_counter() - t0)
            return out
        except vs.HTTPException as e:
            c.labels("failure").inc(); h.labels("failure").observe(time.perf_counter() - t0)
            raise HTTPException(status_code=e.status_code, detail=e.detail)
        except HTTPException:
            c.labels("failure").inc(); h.labels("failure").observe(time.perf_counter() - t0)
            raise
        except Exception as e:
            c.labels("failure").inc(); h.labels("failure").observe(time.perf_counter() - t0)
            raise HTTPException(status_code=500, detail=str(e))

    @app.get("/metrics")
    async def metrics():
        return Response(generate_latest(reg), media_type=CONTENT_TYPE_LATEST)

    @app.get("/health", response_model=HealthStatus)
    def health_check():
        if app.state.store is None:
            raise HTTPException(status_code=500, detail="RAG operations not initialized")
        return HealthStatus(status="Healthy")

    @app.post("/index", response_model=list[Document])
    def index_documents(request: IndexRequest):   # main.py:250-272
        def go():
            docs = [{"text": d.text, "metadata": d.metadata or {}} for d in request.documents]
            t0 = time.perf_counter()
            ids = store.index_documents(request.index_name, docs)
            emb_lat.labels("success", emb_mode).observe(time.perf_counter() - t0)
            emb_cnt.labels("success", emb_mode).inc()
            return [Document(doc_id=i, text=d.text, metadata=d.metadata) for i, d in zip(ids, request.documents)]
        return run("index", go)

    @app.post("/retrieve", response_model=RetrieveResponse)
    async def retrieve_from_index(request: RetrieveRequest):   # main.py:742-771
        """one query per request on the wire, as in the reference; concurrent requests are coalesced into one batched engine
        call (the corpus is streamed once per batch, not once per request) -- the handler itself never blocks the loop"""
        import asyncio
        h, c = M["retrieve"]
        t0 = time.perf_counter()
        try:
            if batcher is not None and batcher.enabled:
                out = await asyncio.wrap_future(batcher.submit(request.index_name, request.query, request.max_node_count,
                                                               request.metadata_filter))
            else:
                out = await asyncio.to_thread(store.retrieve, request.index_name, request.query, request.max_node_count,
                                              request.metadata_filter)
            res_count.observe(out["count"])
            vs_lat.labels("query", "success").observe(getattr(store, "last_retrieve_seconds", 0.0))
            scores = [r["score"] for r in out["results"]]
            if scores:
                low_score.observe(min(scores)); avg_score.observe(sum(scores) / len(scores))
            c.labels("success").inc(); h.labels("success").observe(time.perf_counter() - t0)
            # models.NodeWithScore on the wire (the three optional scores serialise as null when unset) without a second
            # pydantic pass over every result: the dicts come from our own store, the schema is fixed
            for r in out["results"]:
                r.setdefault("dense_score", None); r.setdefault("sparse_score", None); r.setdefault("source", None)
                r.setdefault("metadata", None)
            return _JSON(out)
        except vs.HTTPException as e:
            c.labels("failure").inc(); h.labels("failure").observe(time.perf_counter() - t0)
            raise HTTPException(status_code=e.status_code, detail=e.detail)
        except HTTPException:
            c.labels("failure").inc(); h.labels("failure").observe(time.perf_counter() - t0)
            raise
        except Exception as e:
            c.labels("failure").inc(); h.labels("failure").observe(time.perf_counter() - t0)
            raise HTTPException(status_code=500, detail=str(e))

    @app.post("/v1/chat/completions")
    def chat_completions(request: dict):   # main.py:326-353; RAG or pass-through: kaito_b200/chat.py
        if llm is None:
            M["chat"][1].labels("failure").inc()
            raise HTTPException(status_code=503, detail="LLM inference URL is not configured; chat completions are unavailable. "
                                                        "Use /retrieve for retrieval-only deployments.")
        return run("chat", lambda: store.chat_completion(request, llm, chat_cfg))

    @app.get("/indexes", response_model=list[str])
    def list_indexes():
        return run("indexes", store.list_indexes)

    @app.get("/indexes/{index_name}/documents", response_model=ListDocumentsResponse)
    def list_documents(index_name: str, limit: int = Query(10, ge=1, le=100), offset: int = Query(0, ge=0),
                       max_text_length: int | None = Query(1000, ge=1), metadata_filter: str | None = Query(None)):
        def go():
            mf = None
            if metadata_filter:
                try:
                    mf = json.loads(metadata_filter)
                except json.JSONDecodeError:
                    raise HTTPException(status_code=400, detail="Invalid metadata filter format. Must be a valid JSON string.")
            return store.list_documents_in_index(unquote(index_name), limit, offset, max_text_length, mf)
        return run("documents", go)

    @app.post("/indexes/{index_name}/documents", response_model=UpdateDocumentResponse)
    def update_documents(index_name: str, request: UpdateDocumentRequest):
        return run("update", lambda: store.update_documents(unquote(index_name), [d.model_dump() for d in request.documents]))

    @app.post("/indexes/{index_name}/documents/delete", response_model=DeleteDocumentResponse)
    def delete_documents(index_name: str, request: DeleteDocumentRequest):
        return run("delete_doc", lambda: store.delete_documents(unquote(index_name), request.doc_ids))

    @app.post("/persist/{index_name}")
    def persist_index(index_name: str, path: str | None = Query(None)):   # main.py:619-649
        def go():
            p = path or os.path.join(cfg["persist_dir"], index_name)
            store.persist(unquote(index_name), p)
            return {"message": f"Successfully persisted index {index_name} to {p}."}
        return run("persist", go)

    @app.post("/load/{index_name}")
    def load_index(index_name: str, path: str | None = Query(None), overwrite: bool = Query(False)):   # main.py:675-701
        def go():
            p = path or os.path.join(cfg["persist_dir"], index_name)
            store.load(unquote(index_name), p, overwrite)
            return {"message": f"Successfully loaded index {index_name} from {p}."}
        return run("load", go)

    @app.delete("/indexes/{index_name}")
    def delete_index(index_name: str):
        def go():
            store.delete_index(unquote(index_name))
            return {"message": f"Successfully deleted index {index_name}."}
        return run("delete", go)

    return app


def resolve_model_dir(model_id: str) -> str | None:
    """A local Hugging Face snapshot of `model_id` (config.json + vocab.txt + weights): the path itself, KRAG_MODEL_DIR,
    or the hub cache layout the reference image pre-populates ($HF_HOME/hub/models--ORG--NAME/snapshots/<rev>)."""
    import glob
    cands = [os.getenv("KRAG_MODEL_DIR"), model_id]
    hf_home = os.getenv("HF_HOME") or os.path.join(os.path.expanduser("~"), ".cache", "huggingface")
    cands += sorted(glob.glob(os.path.join(hf_home, "hub", "models--" + model_id.replace("/", "--"), "snapshots", "*")), reverse=True)
    for c in cands:
        if c and os.path.isfile(os.path.join(c, "config.json")) and os.path.isfile(os.path.join(c, "vocab.txt")):
            return c
    return None


def _gpu_count() -> int:
    try:
        import torch
        return int(torch.cuda.device_count())
    except Exception:
        return 1


def main():
    """entry point of the image's `python3 main.py` shim (preset_rag.go:186): port 5000, /health probes."""
    import sys
    import uvicorn
    from . import _native
    from .embedding import GpuBertEmbedding, HashingEmbedding, read_snapshot_spec
    # the event loop thread and the coalescer's dispatcher thread share the GIL; the dispatcher re-acquires it after every
    # engine (ctypes) call, and with the default 5 ms switch interval each re-acquisition can wait that long behind a busy loop
    sys.setswitchinterval(float(os.getenv("KRAG_GIL_SWITCH_S", "0.0002")))
    cfg = env_config()
    if cfg["vector_db_type"] not in ("faiss", "krag"):
        raise SystemExit(f"VECTOR_DB_TYPE={cfg['vector_db_type']} is not served by this image (faiss-compatible engine only)")
    source = cfg["embedding_source"].lower()
    if source not in ("local", "remote"):
        raise SystemExit("Invalid Embedding Type Specified (Must be Local or Remote)")          # main.py:133-141
    model_dir = resolve_model_dir(cfg["embedding_model"]) if source == "local" else None
    if model_dir:
        try:
            read_snapshot_spec(model_dir)            # refuse a snapshot K5 cannot run before any GPU work starts
        except ValueError as e:
            raise SystemExit(f"embedding model '{cfg['embedding_model']}' is not supported by this image: {e}")
    rerank_dir = os.getenv("KRAG_RERANK_MODEL_DIR") or None
    if rerank_dir:
        from .rerank import is_colbert_snapshot, precision_from_env, read_colbert_spec, read_cross_encoder_spec, store_bytes_from_env
        try:
            # refuse a reranker K5 cannot run before any GPU work starts
            colbert = is_colbert_snapshot(rerank_dir)
            (read_colbert_spec if colbert else read_cross_encoder_spec)(rerank_dir)
            rerank_precision = precision_from_env()
            rerank_store = store_bytes_from_env(colbert)
            if int(os.getenv("KRAG_RERANK_CANDIDATES", "30")) < 1:
                raise ValueError("KRAG_RERANK_CANDIDATES must be >= 1")
        except ValueError as e:
            raise SystemExit(f"reranker '{rerank_dir}' is not supported by this image: {e}")
    n_gpus = int(os.getenv("KRAG_NUM_GPUS", "0")) or _gpu_count()
    ctx = _native.Context(device_id=cfg["device_id"], rank=0, world_size=max(1, n_gpus),
                          row_storage=_native.row_storage_from_env())
    engine, workers = ctx, []
    if n_gpus > 1:
        # one replica per RAGEngine (manifests.go:81): every GPU of the pod belongs to this service.  Rank 0 (this process)
        # serves HTTP and shard 0; one worker process per extra GPU holds the other shards (kaito_b200/sharded_engine.py)
        import socket
        import torch
        from . import sharded_engine as se
        with socket.socket() as sk:
            sk.bind(("127.0.0.1", 0))
            port = sk.getsockname()[1]
        workers = se.spawn_workers(n_gpus, port)
        ctl = se.init_distributed(0, n_gpus, cfg["device_id"], port)
        engine = se.ShardedEngine(se.native_stages_factory(ctx), torch.device("cuda", cfg["device_id"]), None, ctl)
    if source == "remote":
        from .embedding import RemoteEmbeddingModel
        embed = RemoteEmbeddingModel(cfg["remote_embedding_url"], cfg["remote_embedding_access_secret"])
    elif model_dir:
        embed = GpuBertEmbedding.from_pretrained(ctx, model_dir)             # K5: BERT forward on the GPU
    elif os.getenv("KRAG_ALLOW_HASHING_EMBEDDING") == "1":
        embed = HashingEmbedding(384)                                        # functional tests only, not a language model
    else:
        raise SystemExit(f"embedding model '{cfg['embedding_model']}' not found locally (no network in the pod): mount a "
                         "Hugging Face snapshot and set KRAG_MODEL_DIR, or KRAG_ALLOW_HASHING_EMBEDDING=1 for functional tests")
    reranker = None
    if rerank_dir:
        from .rerank import GpuCrossEncoder, GpuLateInteractionReranker, is_colbert_snapshot
        try:
            # on rank 0 after the exchange: K5 + MaxSim (ColBERT) or K5 + classifier head (cross-encoder)
            if is_colbert_snapshot(rerank_dir):
                reranker = GpuLateInteractionReranker.from_pretrained(ctx, rerank_dir, precision=rerank_precision, store_bytes=rerank_store)
            else:
                reranker = GpuCrossEncoder.from_pretrained(ctx, rerank_dir, precision=rerank_precision)
        except ValueError as e:
            raise SystemExit(f"reranker '{rerank_dir}' is not supported by this image: {e}")
    app = create_app(vs.VectorStore(embed, engine, reranker=reranker), cfg)
    fronts, rpc = [], None
    try:
        n_front = int(os.getenv("KRAG_HTTP_WORKERS", "0"))
        if n_front > 0 and app.state.batcher is not None and app.state.batcher.enabled:
            # N front-end processes own the public port; this process keeps the engine, the coalescer and the full API on a
            # loopback port the workers proxy to (kaito_b200/frontend.py, kaito_b200/rpc.py)
            import tempfile
            from . import frontend
            from .rpc import RetrieveRpcServer
            engine_port = int(os.getenv("KRAG_ENGINE_PORT", "5001"))
            rpc = RetrieveRpcServer(app.state.batcher, app.state.observe_retrieve, (vs.HTTPException, HTTPException),
                                    path=os.path.join(tempfile.gettempdir(), f"krag-rpc-{os.getpid()}.sock"))
            fronts = frontend.spawn(n_front, "0.0.0.0", 5000, f"127.0.0.1:{engine_port}", rpc.path, None, RAG_MAX_TOP_K)
            uvicorn.run(app, host="127.0.0.1", port=engine_port)
        else:
            uvicorn.run(app, host="0.0.0.0", port=5000)
    finally:
        for p in fronts:
            p.terminate()
        if rpc is not None:
            rpc.close()
        if workers:
            engine.shutdown()
            for w in workers:
                w.wait(timeout=30)


if __name__ == "__main__":
    main()
