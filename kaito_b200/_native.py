"""ctypes binding of libkaito_rag.so (include/kaito_rag.h).

The CUDA library IS the product path: there is no CPU or PyTorch fallback.  Importing this
module without the built library, or initialising it without an sm_90 (H100) GPU, raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libkaito_rag.so")

KRAG_OK = 0
KRAG_E_INVALID, KRAG_E_NO_DEVICE, KRAG_E_CUDA, KRAG_E_OOM = -1, -2, -3, -4
KRAG_E_NOT_FOUND, KRAG_E_STATE, KRAG_E_IO, KRAG_E_UNSUPPORTED = -5, -6, -7, -8
KRAG_KEY_PAD = 0xFFFFFFFFFFFFFFFF
KRAG_MAX_TOP_K = 300
KRAG_MAX_POOL = 1024
FUSION_REFERENCE, FUSION_SIMILARITY = 0, 1
FILTER_PUSHDOWN = 0x100   # OR into fusion_mode: the allow bitmap restricts the dense and BM25 scans themselves
DENSE_AUTO, DENSE_SCAN, DENSE_TC, DENSE_TC_BF16, DENSE_TC_TF32 = 0, 1, 2, 3, 4
ROWS_DEVICE, ROWS_HOST = 0, 1   # krag_config.row_storage: fp32 rows in HBM, or in pinned host memory with a bf16 device copy
POOL_CLS, POOL_MEAN = 0, 1      # krag_embedder_set_pooling: the [CLS] row, or the mean over every token of the sequence

# every symbol include/kaito_rag.h declares (tests check the export table against this)
SYMBOLS = [
    "krag_version", "krag_last_error", "krag_init", "krag_shutdown", "krag_launch_count", "krag_device_bytes", "krag_ctx_stream",
    "krag_index_create", "krag_index_drop", "krag_index_reserve", "krag_index_add", "krag_index_remove",
    "krag_index_commit", "krag_index_commit_local", "krag_index_commit_global", "krag_index_stats",
    "krag_index_node_ids", "krag_index_set_ordinal_map", "krag_index_persist", "krag_index_load", "krag_search_dense", "krag_search_bm25",
    "krag_retrieve", "krag_dev_dense_candidates", "krag_dev_bm25_candidates", "krag_dev_merge", "krag_dev_fuse",
    "krag_synth_fill", "krag_index_read_rows", "krag_index_read_postings", "krag_tc_fallback_queries",
    "krag_debug_tc_dump", "krag_debug_read_stored_rows", "krag_last_dense_kernel", "krag_embedder_create", "krag_embedder_load_tensor",
    "krag_embedder_finalize", "krag_embed", "krag_embed_dev", "krag_embedder_destroy", "krag_debug_gemm_tf32",
    "krag_debug_linear_ln", "krag_index_set_dense_mode", "krag_text_analyze", "krag_wordpiece_create",
    "krag_wordpiece_encode_batch", "krag_wordpiece_destroy", "krag_p2p_create", "krag_p2p_connect", "krag_dev_exchange_merge", "krag_p2p_destroy",
    "krag_host_pinned_bytes", "krag_host_rows_fetched", "krag_index_compact", "krag_last_compact",
    "krag_last_commit", "krag_index_alive_bitmap", "krag_redeal_begin", "krag_redeal_tables", "krag_redeal_prepare",
    "krag_dev_redeal_pack", "krag_dev_redeal_unpack", "krag_redeal_finish", "krag_redeal_abort", "krag_embedder_set_pooling",
    "krag_debug_embedder_cls_rows", "krag_rerank", "krag_embedder_set_precision", "krag_debug_gemm_f16",
    "krag_embedder_set_position_offset", "krag_text_unigram_create", "krag_text_unigram_encode_batch",
    "krag_text_unigram_destroy", "krag_debug_tc_dump_pass", "krag_debug_tc_prune", "krag_debug_relative_bucket",
    "krag_wordpiece_create_specials", "krag_embedder_set_rotary", "krag_debug_rotary_cos_sin",
    "krag_embedder_set_late_interaction", "krag_late_rerank", "krag_debug_late_vectors",
    "krag_embedder_set_store_budget", "krag_late_store_create", "krag_late_store_destroy", "krag_late_store_append",
    "krag_late_store_truncate", "krag_late_store_compact", "krag_late_store_stats", "krag_late_rerank_stored",
    "krag_debug_late_store_vectors",
]
# krag_debug_tc_dump_pass / krag_debug_tc_prune: the prune pass to run (KRAG_TC_PASS_*)
TC_PASS_TF32, TC_PASS_BF16_SPLIT, TC_PASS_BF16_SHADOW, TC_PASS_BF16_HOST = 0, 1, 2, 3
# krag_embedder_set_precision: split-fp16 products held to fp32 arithmetic, or fp16 operands with fp32 accumulation
PRECISIONS = {"fp32": 0, "fp16": 1}
RERANK_SIGMOID, RERANK_IDENTITY = 0, 1   # krag_rerank: activation of the classifier logit


class KragError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libkaito_rag error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("device_id", C.c_int32), ("rank", C.c_int32), ("world_size", C.c_int32), ("dense_mode", C.c_int32),
                ("search_slots", C.c_int32), ("row_storage", C.c_int32), ("reserved", C.c_int32 * 2)]


class Stats(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_live", C.c_int64), ("nnz", C.c_int64), ("n_docs_global", C.c_int64),
                ("total_len_global", C.c_int64), ("vocab", C.c_int64), ("ordinal_base", C.c_int64), ("dim", C.c_int32),
                ("dim_padded", C.c_int32), ("committed", C.c_int32), ("reserved", C.c_int32),
                ("device_bytes", C.c_int64)]


class BertConfig(C.Structure):
    _fields_ = [("layers", C.c_int32), ("hidden", C.c_int32), ("heads", C.c_int32), ("intermediate", C.c_int32),
                ("vocab", C.c_int32), ("max_position", C.c_int32), ("type_vocab", C.c_int32), ("ln_eps", C.c_float)]


_lib = None


def load() -> C.CDLL:
    """dlopen the in-tree library; fail loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(make -C kaito_b200/csrc). kaito_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, u32, f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_double
    L.krag_version.restype = i32
    L.krag_last_error.restype = C.c_char_p
    L.krag_init.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    L.krag_shutdown.argtypes = [vp]
    L.krag_launch_count.argtypes = [vp]
    L.krag_launch_count.restype = i64
    L.krag_device_bytes.restype = i64
    L.krag_host_pinned_bytes.restype = i64
    L.krag_host_rows_fetched.restype = i64
    L.krag_ctx_stream.argtypes = [vp]
    L.krag_ctx_stream.restype = vp
    L.krag_index_create.argtypes = [vp, C.c_char_p, i32, C.POINTER(vp)]
    L.krag_index_drop.argtypes = [vp]
    L.krag_index_reserve.argtypes = [vp, i64, i64]
    L.krag_index_add.argtypes = [vp, i64, vp, vp, vp, vp, vp, vp]
    L.krag_index_remove.argtypes = [vp, i64, vp, C.POINTER(i64)]
    L.krag_index_compact.argtypes = [vp, C.POINTER(i64)]
    L.krag_index_alive_bitmap.argtypes = [vp, vp, i64, C.POINTER(i64)]
    L.krag_redeal_begin.argtypes = [vp, vp, i64, i64, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)]
    L.krag_redeal_tables.argtypes = [vp, vp, vp, vp]
    L.krag_redeal_prepare.argtypes = [vp, vp]
    L.krag_dev_redeal_pack.argtypes = [vp, i64, vp, vp, vp]
    L.krag_dev_redeal_unpack.argtypes = [vp, i64, vp, vp, vp]
    L.krag_redeal_finish.argtypes = [vp, vp, C.POINTER(i64)]
    L.krag_redeal_abort.argtypes = [vp]
    L.krag_index_commit.argtypes = [vp, i64]
    L.krag_index_commit_local.argtypes = [vp, i64, vp, C.POINTER(i64), C.POINTER(i64)]
    L.krag_index_commit_global.argtypes = [vp, i64, vp, i64, i64, i64]
    L.krag_index_stats.argtypes = [vp, C.POINTER(Stats)]
    L.krag_index_set_ordinal_map.argtypes = [vp, i64, i64]
    L.krag_index_node_ids.argtypes = [vp, i64, vp, vp]
    L.krag_index_persist.argtypes = [vp, C.c_char_p]
    L.krag_index_load.argtypes = [vp, C.c_char_p, C.c_char_p, C.POINTER(vp)]
    L.krag_search_dense.argtypes = [vp, i32, vp, i32, vp, vp]
    L.krag_search_bm25.argtypes = [vp, i32, vp, vp, i32, vp, vp]
    L.krag_retrieve.argtypes = [vp, i32, vp, vp, vp, i32, f64, f64, f64, i32, vp, i64, vp, vp, vp, vp, vp, vp]
    L.krag_dev_dense_candidates.argtypes = [vp, i32, vp, i32, vp, vp]
    L.krag_dev_bm25_candidates.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp]
    L.krag_dev_merge.argtypes = [vp, i32, i32, i32, vp, vp, vp]
    L.krag_dev_fuse.argtypes = [vp, i32, i32, i32, vp, vp, f64, f64, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.krag_synth_fill.argtypes = [vp, i64, i64, C.c_uint64, i64]
    L.krag_index_read_rows.argtypes = [vp, i64, i64, vp]
    L.krag_index_read_postings.argtypes = [vp, u32, i64, vp, vp, C.POINTER(i64)]
    L.krag_embedder_create.argtypes = [vp, C.POINTER(BertConfig), C.POINTER(vp)]
    L.krag_embedder_load_tensor.argtypes = [vp, C.c_char_p, vp, i64]
    L.krag_embedder_finalize.argtypes = [vp]
    L.krag_embed.argtypes = [vp, i32, vp, vp, vp]
    L.krag_embed_dev.argtypes = [vp, i32, vp, vp, vp, i32, vp]
    L.krag_embedder_set_pooling.argtypes = [vp, i32]
    L.krag_debug_embedder_cls_rows.argtypes = [vp, i32]
    L.krag_embedder_set_precision.argtypes = [vp, i32]
    L.krag_embedder_set_position_offset.argtypes = [vp, i32]
    L.krag_rerank.argtypes = [vp, i32, vp, vp, vp, vp, i32, i32, vp, vp]
    L.krag_embedder_destroy.argtypes = [vp]
    L.krag_debug_gemm_tf32.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp, i32, vp, i32, i32, C.POINTER(C.c_float)]
    L.krag_debug_gemm_f16.argtypes = L.krag_debug_gemm_tf32.argtypes
    L.krag_debug_linear_ln.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, C.c_float, vp]
    L.krag_index_set_dense_mode.argtypes = [vp, i32, i32]
    L.krag_text_analyze.argtypes = [C.c_char_p, i64, vp, i64, C.POINTER(i64), C.POINTER(i32)]
    L.krag_wordpiece_create.argtypes = [C.c_char_p, i64, i32, C.POINTER(vp)]
    L.krag_wordpiece_create_specials.argtypes = [C.c_char_p, i64, i32, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(vp)]
    L.krag_debug_relative_bucket.argtypes = [i32]
    L.krag_embedder_set_rotary.argtypes = [vp, C.c_float]
    L.krag_debug_rotary_cos_sin.argtypes = [C.c_float, i32, i32, vp, vp]
    L.krag_embedder_set_late_interaction.argtypes = [vp, i32, vp, i64]
    L.krag_late_rerank.argtypes = [vp, i32, i32, vp, vp, i32, vp, vp, vp, vp, vp, i32, vp, vp]
    L.krag_debug_late_vectors.argtypes = [vp, i32, vp, vp, vp, vp]
    L.krag_embedder_set_store_budget.argtypes = [vp, i64]
    L.krag_late_store_create.argtypes = [vp, C.POINTER(vp)]
    L.krag_late_store_destroy.argtypes = [vp]
    L.krag_late_store_append.argtypes = [vp, i32, vp, vp, vp, vp]
    L.krag_late_store_truncate.argtypes = [vp, i64]
    L.krag_late_store_compact.argtypes = [vp, vp, i64]
    L.krag_late_store_stats.argtypes = [vp, vp, vp, vp, vp]
    L.krag_late_rerank_stored.argtypes = [vp, vp, i32, i32, vp, vp, i32, vp, vp, vp, vp, vp, i32, vp, vp]
    L.krag_debug_late_store_vectors.argtypes = [vp, i64, vp, i64]
    L.krag_wordpiece_encode_batch.argtypes = [vp, i64, C.c_char_p, vp, i32, vp, vp]
    L.krag_wordpiece_destroy.argtypes = [vp]
    L.krag_text_unigram_create.argtypes = [C.c_char_p, vp, vp, i64, i32, C.c_char_p, i64, i32, C.c_char_p, vp, vp, vp, i32,
                                           C.POINTER(vp)]
    L.krag_text_unigram_encode_batch.argtypes = [vp, i64, C.c_char_p, vp, i32, vp, vp]
    L.krag_text_unigram_destroy.argtypes = [vp]
    L.krag_p2p_create.argtypes = [vp, i32, i32, i32, i32, C.POINTER(vp), vp]
    L.krag_p2p_connect.argtypes = [vp, vp]
    L.krag_dev_exchange_merge.argtypes = [vp, i32, i32, i32, vp, vp, vp]
    L.krag_p2p_destroy.argtypes = [vp]
    L.krag_tc_fallback_queries.restype = i64
    L.krag_last_dense_kernel.argtypes = [C.POINTER(C.c_float), C.POINTER(i32), C.POINTER(i64), C.POINTER(i64)]
    L.krag_last_compact.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(i64), C.POINTER(i64)]
    L.krag_last_commit.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(i32), C.POINTER(i64), C.POINTER(i64)]
    L.krag_debug_tc_dump.argtypes = [vp, i32, vp, vp, i64, C.POINTER(i64), C.POINTER(i32)]
    L.krag_debug_tc_dump_pass.argtypes = [vp, i32, i32, vp, vp, i64, C.POINTER(i64), C.POINTER(i32)]
    L.krag_debug_tc_prune.argtypes = [vp, i32, i32, vp, vp, i32, vp, vp]
    L.krag_debug_read_stored_rows.argtypes = [vp, i64, i64, vp]
    for name in SYMBOLS:
        fn = getattr(L, name)
        if fn.restype is C.c_int:  # default: every remaining call returns an int32 status
            fn.restype = i32
    _lib = L
    return L


def check(rc: int):
    if rc != KRAG_OK:
        raise KragError(rc, load().krag_last_error().decode("utf-8", "replace"))


def ptr(a):
    """numpy array / int address / None -> void*"""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(int(a))


def last_dense_kernel():
    """(ms, kernel_id, algorithmic_bytes, flops) of the dominant dense kernel of the last search."""
    ms, kid, by, fl = C.c_float(0), C.c_int32(0), C.c_int64(0), C.c_int64(0)
    check(load().krag_last_dense_kernel(C.byref(ms), C.byref(kid), C.byref(by), C.byref(fl)))
    return ms.value, kid.value, by.value, fl.value


def last_compact() -> dict:
    """figures of the last Index.compact() of this process: move_ms (CUDA events around the row moves), postings_ms,
    rows_moved, bytes_moved (moved rows and term lists, each byte counted once)"""
    mv, po, rows, by = C.c_float(0), C.c_float(0), C.c_int64(0), C.c_int64(0)
    check(load().krag_last_compact(C.byref(mv), C.byref(po), C.byref(rows), C.byref(by)))
    return {"move_ms": mv.value, "postings_ms": po.value, "rows_moved": rows.value, "bytes_moved": by.value}


def last_commit() -> dict:
    """figures of the last commit of this process: total_ms (host clock), host_ms (idf on the host), merged (1: the committed
    postings were merged with the changes, 0: a full build), postings_written, delta_entries (term-list entries read)"""
    tot, host, mg, pw, de = C.c_float(0), C.c_float(0), C.c_int32(0), C.c_int64(0), C.c_int64(0)
    check(load().krag_last_commit(C.byref(tot), C.byref(host), C.byref(mg), C.byref(pw), C.byref(de)))
    return {"total_ms": tot.value, "host_ms": host.value, "merged": mg.value, "postings_written": pw.value,
            "delta_entries": de.value}


def device_bytes() -> int:
    """device memory, in bytes, this process currently holds through the library (every context, index and embedder)"""
    return int(load().krag_device_bytes())


def row_storage_from_env(environ=None) -> int:
    """KRAG_ROW_STORAGE=device|host (default device) -> ROWS_DEVICE / ROWS_HOST; any other value raises ValueError"""
    v = (os.environ if environ is None else environ).get("KRAG_ROW_STORAGE", "device").strip().lower()
    if v not in ("device", "host"):
        raise ValueError(f"KRAG_ROW_STORAGE={v!r}: expected 'device' or 'host'")
    return ROWS_HOST if v == "host" else ROWS_DEVICE


def host_pinned_bytes() -> int:
    """pinned host memory, in bytes, this process currently holds through the library (ROWS_HOST rows)"""
    return int(load().krag_host_pinned_bytes())


def host_rows_fetched() -> int:
    """rows rescored from host memory by ROWS_HOST searches so far (process-wide)"""
    return int(load().krag_host_rows_fetched())


class Context:
    """krag_ctx: one per process per GPU.  row_storage applies to every index created or loaded in the context."""

    def __init__(self, device_id: int = 0, rank: int = 0, world_size: int = 1, dense_mode: int = DENSE_AUTO,
                 search_slots: int = 0, row_storage: int = ROWS_DEVICE):
        L = load()
        cfg = Config(device_id=device_id, rank=rank, world_size=world_size, dense_mode=dense_mode,
                     search_slots=search_slots, row_storage=row_storage)
        h = C.c_void_p()
        check(L.krag_init(C.byref(cfg), C.byref(h)))
        self._h, self._L = h, L
        self.device_id, self.rank, self.world_size = device_id, rank, world_size

    def close(self):
        if self._h:
            check(self._L.krag_shutdown(self._h))
            self._h = None

    def launch_count(self) -> int:
        return int(self._L.krag_launch_count(self._h))

    def stream(self) -> int:
        return int(self._L.krag_ctx_stream(self._h) or 0)

    def create_index(self, name: str, dim: int) -> "Index":
        h = C.c_void_p()
        check(self._L.krag_index_create(self._h, name.encode(), dim, C.byref(h)))
        return Index(self, h, name, dim)

    def load_index(self, name: str, path: str) -> "Index":
        h = C.c_void_p()
        check(self._L.krag_index_load(self._h, name.encode(), path.encode(), C.byref(h)))
        ix = Index(self, h, name, 0)
        ix.dim = ix.stats().dim
        return ix

    # ---- device-pointer stage API (multi-GPU host) ----
    def dev_merge(self, n_lists, batch, P, d_in, d_out, stream=0):
        check(self._L.krag_dev_merge(self._h, n_lists, batch, P, ptr(d_in), ptr(d_out), ptr(stream)))

    def dev_fuse(self, batch, P, k, d_dense, d_bm25, vw, tw, mode, d_allow, d_final, d_dense_out, d_sparse_out, d_rank,
                 d_ord, d_count, stream=0):
        check(self._L.krag_dev_fuse(self._h, batch, P, k, ptr(d_dense), ptr(d_bm25), vw, tw, mode, ptr(d_allow),
                                    ptr(d_final), ptr(d_dense_out), ptr(d_sparse_out), ptr(d_rank), ptr(d_ord),
                                    ptr(d_count), ptr(stream)))


class P2PExchange:
    """krag_p2p: candidate-list all-gather + merge over NVLink peer memory (our kernels, not NCCL)."""

    def __init__(self, ctx: "Context", rank: int, world: int, max_batch: int, max_P: int):
        self._L = ctx._L
        h = C.c_void_p()
        self.handle = np.zeros(64, np.uint8)
        check(self._L.krag_p2p_create(ctx._h, rank, world, max_batch, max_P, C.byref(h), ptr(self.handle)))
        self._h, self.world = h, world

    def connect(self, handles: np.ndarray):
        handles = np.ascontiguousarray(handles, np.uint8).reshape(self.world, 64)
        check(self._L.krag_p2p_connect(self._h, ptr(handles)))

    def exchange_merge(self, n_lists, batch, P, d_local, d_merged, stream=0):
        check(self._L.krag_dev_exchange_merge(self._h, n_lists, batch, P, ptr(d_local), ptr(d_merged), ptr(stream)))

    def destroy(self):
        if self._h:
            check(self._L.krag_p2p_destroy(self._h))
            self._h = None


class Embedder:
    """krag_embedder: BERT-family encoder forward on the GPU (K5).  Variants (kaito_rag.h): MPNet when loaded with
    encoder.relative_attention_bias.weight; nomic-bert's rotary positions with set_rotary(base) before load_state_dict; a
    gated (SwiGLU) FFN when loaded with encoder.layer.{l}.intermediate.gate.weight / .bias on every layer."""

    def __init__(self, ctx: "Context", layers, hidden, heads, intermediate, vocab, max_position=512, type_vocab=2,
                 ln_eps=1e-12):
        self.ctx, self._L, self.hidden = ctx, ctx._L, hidden
        cfg = BertConfig(layers, hidden, heads, intermediate, vocab, max_position, type_vocab, ln_eps)
        h = C.c_void_p()
        check(self._L.krag_embedder_create(ctx._h, C.byref(cfg), C.byref(h)))
        self._h = h

    def load_state_dict(self, state: dict, head: bool = False):
        """state: Hugging Face BertModel names -> numpy fp32 arrays (position_ids entries are ignored).  head=False: pooler
        and classifier entries are ignored too; head=True: they are loaded, and rerank() may be called"""
        for name, arr in state.items():
            if name.endswith("position_ids") or (not head and name.startswith(("pooler.", "classifier."))):
                continue
            a = np.ascontiguousarray(arr, np.float32)
            check(self._L.krag_embedder_load_tensor(self._h, name.encode(), ptr(a), a.size))
        check(self._L.krag_embedder_finalize(self._h))

    def embed(self, token_lists) -> np.ndarray:
        offs = np.zeros(len(token_lists) + 1, np.int32)
        for i, t in enumerate(token_lists):
            offs[i + 1] = offs[i] + len(t)
        flat = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in token_lists]), np.int32)
        out = np.empty((len(token_lists), self.hidden), np.float32)
        check(self._L.krag_embed(self._h, len(token_lists), ptr(flat), ptr(offs), ptr(out)))
        return out

    def embed_flat(self, flat_tokens: np.ndarray, offsets: np.ndarray) -> np.ndarray:
        """embed() for tokens that are already packed (int32 ids, int32 offsets [batch + 1])"""
        flat_tokens = np.ascontiguousarray(flat_tokens, np.int32); offsets = np.ascontiguousarray(offsets, np.int32)
        out = np.empty((len(offsets) - 1, self.hidden), np.float32)
        check(self._L.krag_embed(self._h, len(offsets) - 1, ptr(flat_tokens), ptr(offsets), ptr(out)))
        return out

    @staticmethod
    def pack(token_lists):
        offs = np.zeros(len(token_lists) + 1, np.int32)
        for i, t in enumerate(token_lists):
            offs[i + 1] = offs[i] + len(t)
        return np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in token_lists]), np.int32), offs

    def embed_dev(self, flat_tokens: np.ndarray, offsets: np.ndarray, d_out: int, ld_out: int, stream: int = 0):
        """embeddings written to device memory (row stride ld_out floats); `stream` waits for them"""
        check(self._L.krag_embed_dev(self._h, len(offsets) - 1, ptr(flat_tokens), ptr(offsets), ptr(d_out), ld_out, ptr(stream)))

    def set_pooling(self, mode: int):
        """POOL_CLS (default) or POOL_MEAN for the following forwards"""
        check(self._L.krag_embedder_set_pooling(self._h, mode))

    def set_precision(self, precision: str):
        """"fp32" (default) or "fp16" for the following forwards (krag_embedder_set_precision)"""
        if precision not in PRECISIONS:
            raise ValueError(f"precision {precision!r}: expected 'fp32' or 'fp16'")
        check(self._L.krag_embedder_set_precision(self._h, PRECISIONS[precision]))

    def set_position_offset(self, off: int):
        """position row of every sequence's first token (krag_embedder_set_position_offset; XLM-R: pad_token_id + 1)"""
        check(self._L.krag_embedder_set_position_offset(self._h, off))

    def set_rotary(self, base: float):
        """rotary positions with this base (nomic-bert: rotary_emb_base 1000) instead of a position table, 0 = off
        (krag_embedder_set_rotary); before load_state_dict, which finalizes"""
        check(self._L.krag_embedder_set_rotary(self._h, float(base)))

    def rerank(self, pair_offsets, flat_tokens, tok_offsets, seg_b, top_k: int, activation: int = RERANK_SIGMOID):
        """krag_rerank: (positions int32 [n_queries, top_k], scores float32 [n_queries, top_k]); -1 / NaN past a query's
        pair count.  seg_b None: unsegmented pairs (token type 0 throughout)"""
        pair_offsets = np.ascontiguousarray(pair_offsets, np.int32)
        flat_tokens = np.ascontiguousarray(flat_tokens, np.int32); tok_offsets = np.ascontiguousarray(tok_offsets, np.int32)
        seg_b = None if seg_b is None else np.ascontiguousarray(seg_b, np.int32)
        nq = len(pair_offsets) - 1
        pos = np.empty((nq, top_k), np.int32)
        sc = np.empty((nq, top_k), np.float32)
        check(self._L.krag_rerank(self._h, nq, ptr(pair_offsets), ptr(flat_tokens), ptr(tok_offsets), ptr(seg_b), activation, top_k,
                                  ptr(pos), ptr(sc)))
        return pos, sc

    def set_late_interaction(self, weight):
        """the ColBERT projection linear.weight [dim, hidden] (no bias) every token row maps through before its L2
        normalisation (krag_embedder_set_late_interaction); before load_state_dict, which finalizes"""
        w = np.ascontiguousarray(weight, np.float32)
        self.li_dim = int(w.shape[0])
        check(self._L.krag_embedder_set_late_interaction(self._h, self.li_dim, ptr(w), w.size))

    def late_rerank(self, q_tokens, q_keys, p_tokens, p_offsets, p_keep, pair_offsets, pair_passage, top_k: int):
        """krag_late_rerank: q_tokens int32 [n_queries, query_len], q_keys [n_queries]; packed passages with their uint8 keep
        mask; pair_passage [n_pairs] indexes the passages.  (positions int32 [n_queries, top_k], scores float32 [n_queries,
        top_k]); -1 / NaN past a query's pair count"""
        q_tokens = np.ascontiguousarray(q_tokens, np.int32)
        nq, ql = q_tokens.shape
        q_keys = np.ascontiguousarray(q_keys, np.int32)
        p_tokens = np.ascontiguousarray(p_tokens, np.int32); p_offsets = np.ascontiguousarray(p_offsets, np.int32)
        p_keep = np.ascontiguousarray(p_keep, np.uint8)
        pair_offsets = np.ascontiguousarray(pair_offsets, np.int32); pair_passage = np.ascontiguousarray(pair_passage, np.int32)
        pos = np.empty((nq, top_k), np.int32)
        sc = np.empty((nq, top_k), np.float32)
        check(self._L.krag_late_rerank(self._h, nq, ql, ptr(q_tokens), ptr(q_keys), len(p_offsets) - 1, ptr(p_tokens), ptr(p_offsets),
                                       ptr(p_keep), ptr(pair_offsets), ptr(pair_passage), top_k, ptr(pos), ptr(sc)))
        return pos, sc

    def debug_late_vectors(self, flat_tokens, offsets, key_lens=None) -> np.ndarray:
        """the unit token vectors [tokens, dim] of packed sequences (krag_debug_late_vectors); key_lens None: every row a key"""
        flat_tokens = np.ascontiguousarray(flat_tokens, np.int32); offsets = np.ascontiguousarray(offsets, np.int32)
        kl = None if key_lens is None else np.ascontiguousarray(key_lens, np.int32)
        out = np.empty((int(offsets[-1]), self.li_dim), np.float32)
        check(self._L.krag_debug_late_vectors(self._h, len(offsets) - 1, ptr(flat_tokens), ptr(offsets), ptr(kl), ptr(out)))
        return out

    def set_store_budget(self, nbytes: int):
        """device bytes every LateStore of this embedder may hold in all (krag_embedder_set_store_budget; 0: none)"""
        check(self._L.krag_embedder_set_store_budget(self._h, int(nbytes)))

    def late_rerank_stored(self, store: "LateStore", q_tokens, q_keys, p_tokens, p_offsets, p_keep, pair_offsets, pair_source,
                           top_k: int):
        """krag_late_rerank_stored: late_rerank with pair_source[j] >= 0 a stored ordinal of `store`, < 0 passage
        ~pair_source[j] of the call (the packed passages may be empty)"""
        q_tokens = np.ascontiguousarray(q_tokens, np.int32)
        nq, ql = q_tokens.shape
        q_keys = np.ascontiguousarray(q_keys, np.int32)
        p_tokens = np.ascontiguousarray(p_tokens, np.int32); p_offsets = np.ascontiguousarray(p_offsets, np.int32)
        p_keep = np.ascontiguousarray(p_keep, np.uint8)
        pair_offsets = np.ascontiguousarray(pair_offsets, np.int32); pair_source = np.ascontiguousarray(pair_source, np.int32)
        pos = np.empty((nq, top_k), np.int32)
        sc = np.empty((nq, top_k), np.float32)
        n_pass = max(len(p_offsets) - 1, 0)
        check(self._L.krag_late_rerank_stored(self._h, store._h, nq, ql, ptr(q_tokens), ptr(q_keys), n_pass, ptr(p_tokens) if n_pass else None,
                                              ptr(p_offsets) if n_pass else None, ptr(p_keep) if n_pass else None, ptr(pair_offsets),
                                              ptr(pair_source), top_k, ptr(pos), ptr(sc)))
        return pos, sc

    def debug_cls_rows(self, on: bool):
        """test hook: False runs the last layer over every token under CLS pooling too (same embeddings)"""
        check(self._L.krag_debug_embedder_cls_rows(self._h, 1 if on else 0))

    def destroy(self):
        if self._h:
            check(self._L.krag_embedder_destroy(self._h))
            self._h = None


class LateStore:
    """krag_late_store: the kept token vectors of passages, per ordinal, on the embedder's GPU (see kaito_rag.h).  Holds its
    embedder, which cannot be destroyed before it."""

    def __init__(self, emb: Embedder):
        self.emb, self._L = emb, emb._L
        h = C.c_void_p()
        check(self._L.krag_late_store_create(emb._h, C.byref(h)))
        self._h = h

    def append(self, p_tokens, p_offsets, p_keep) -> np.ndarray:
        """the next len(p_offsets) - 1 ordinals; uint8 [n]: 1 where the passage was stored"""
        p_tokens = np.ascontiguousarray(p_tokens, np.int32); p_offsets = np.ascontiguousarray(p_offsets, np.int32)
        p_keep = np.ascontiguousarray(p_keep, np.uint8)
        out = np.zeros(len(p_offsets) - 1, np.uint8)
        check(self._L.krag_late_store_append(self._h, len(out), ptr(p_tokens), ptr(p_offsets), ptr(p_keep), ptr(out)))
        return out

    def truncate(self, n_ordinals: int):
        check(self._L.krag_late_store_truncate(self._h, int(n_ordinals)))

    def compact(self, alive: np.ndarray):
        """alive: bool [ordinals]; the live ordinals keep their order and become 0 .. n_live - 1"""
        alive = np.asarray(alive, bool)
        bm = np.zeros((len(alive) + 31) // 32, np.uint32)
        idx = np.flatnonzero(alive)
        np.bitwise_or.at(bm, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
        check(self._L.krag_late_store_compact(self._h, ptr(bm), len(alive)))

    def stats(self) -> dict:
        v = [C.c_int64() for _ in range(4)]
        check(self._L.krag_late_store_stats(self._h, *[C.byref(x) for x in v]))
        return dict(zip(("ordinals", "stored", "rows", "device_bytes"), (int(x.value) for x in v)))

    def debug_vectors(self, ordinal: int, n_rows: int) -> np.ndarray:
        out = np.empty((n_rows, self.emb.li_dim), np.float32)
        check(self._L.krag_debug_late_store_vectors(self._h, int(ordinal), ptr(out), int(n_rows)))
        return out

    def destroy(self):
        if self._h:
            check(self._L.krag_late_store_destroy(self._h))
            self._h = None


def debug_relative_bucket(rel: int) -> int:
    """the MPNet relative-position bucket K5's attention applies at rel = key - query (krag_debug_relative_bucket; no GPU)"""
    return int(load().krag_debug_relative_bucket(rel))


def debug_rotary_cos_sin(base: float, dh: int, pos: int) -> tuple[np.ndarray, np.ndarray]:
    """the fp32 (cos [dh / 2], sin [dh / 2]) a rotary embedder applies at position pos (krag_debug_rotary_cos_sin; no GPU)"""
    cos, sin = np.empty(dh // 2, np.float32), np.empty(dh // 2, np.float32)
    check(load().krag_debug_rotary_cos_sin(float(base), dh, pos, ptr(cos), ptr(sin)))
    return cos, sin


def debug_gemm_tf32(ctx: "Context", A, B, bias, residual=None, gelu=False, tile_n=0) -> np.ndarray:
    """tile_n = 0: the tiles the forward picks for this shape; 32 / 64 / 128: 128 x tile_n tiles, whole K range"""
    return _debug_gemm(ctx, A, B, bias, residual, gelu, tile_n, 0)[0]


def debug_gemm_f16(ctx: "Context", A, B, bias, residual=None, gelu=False, tile_n=0) -> np.ndarray:
    """the single-plane fp16 GEMM of the fp16 precision mode (A and B rounded to fp16, fp32 accumulation); tile_n as above, or 256"""
    return _debug_gemm(ctx, A, B, bias, residual, gelu, tile_n, 0, "krag_debug_gemm_f16")[0]


def debug_gemm_time(ctx: "Context", A, B, bias, residual=None, gelu=False, tile_n=0, reps=50, f16=False):
    """(C, mean ms of one GEMM launch over `reps` launches on the device operands); f16: the single-plane fp16 GEMM"""
    return _debug_gemm(ctx, A, B, bias, residual, gelu, tile_n, reps, "krag_debug_gemm_f16" if f16 else "krag_debug_gemm_tf32")


def _debug_gemm(ctx, A, B, bias, residual, gelu, tile_n, reps, fn="krag_debug_gemm_tf32"):
    A = np.ascontiguousarray(A, np.float32); B = np.ascontiguousarray(B, np.float32)
    bias = np.ascontiguousarray(bias, np.float32)
    if residual is not None:
        residual = np.ascontiguousarray(residual, np.float32)
    out = np.empty((A.shape[0], B.shape[0]), np.float32)
    ms = C.c_float(0.0)
    check(getattr(load(), fn)(ctx._h, A.shape[0], B.shape[0], A.shape[1], ptr(A), ptr(B), ptr(bias), ptr(residual),
                              1 if gelu else 0, ptr(out), int(tile_n), int(reps), C.byref(ms)))
    return out, float(ms.value)


def debug_linear_ln(ctx: "Context", A, B, bias, residual, gamma, beta, eps=1e-12) -> np.ndarray:
    A = np.ascontiguousarray(A, np.float32); B = np.ascontiguousarray(B, np.float32)
    bias = np.ascontiguousarray(bias, np.float32); gamma = np.ascontiguousarray(gamma, np.float32)
    beta = np.ascontiguousarray(beta, np.float32)
    if residual is not None:
        residual = np.ascontiguousarray(residual, np.float32)
    out = np.empty((A.shape[0], B.shape[0]), np.float32)
    check(load().krag_debug_linear_ln(ctx._h, A.shape[0], B.shape[0], A.shape[1], ptr(A), ptr(B), ptr(bias), ptr(residual),
                                      ptr(gamma), ptr(beta), eps, ptr(out)))
    return out


class Index:
    """krag_index: one document shard (dense rows + BM25 postings) resident on one GPU."""

    def __init__(self, ctx: Context, handle, name: str, dim: int):
        self.ctx, self._h, self.name, self.dim = ctx, handle, name, dim
        self._L = ctx._L

    def drop(self):
        if self._h:
            check(self._L.krag_index_drop(self._h))
            self._h = None

    def reserve(self, rows: int, nnz: int = 0):
        check(self._L.krag_index_reserve(self._h, rows, nnz))

    def add(self, node_ids, vecs, term_offsets=None, term_ids=None, term_tf=None, doc_len=None):
        node_ids = np.ascontiguousarray(node_ids, np.uint64)
        vecs = np.ascontiguousarray(vecs, np.float32).reshape(len(node_ids), self.dim)
        if term_offsets is not None:
            term_offsets = np.ascontiguousarray(term_offsets, np.int64)
            term_ids = np.ascontiguousarray(term_ids, np.uint32)
            term_tf = np.ascontiguousarray(term_tf, np.uint16)
            doc_len = np.ascontiguousarray(doc_len, np.uint32)
        check(self._L.krag_index_add(self._h, len(node_ids), ptr(node_ids), ptr(vecs), ptr(term_offsets), ptr(term_ids),
                                     ptr(term_tf), ptr(doc_len)))

    def remove(self, node_ids) -> int:
        node_ids = np.ascontiguousarray(node_ids, np.uint64)
        n = C.c_int64(0)
        check(self._L.krag_index_remove(self._h, len(node_ids), ptr(node_ids), C.byref(n)))
        return n.value

    def compact(self) -> int:
        """remove the tombstoned rows in place; live rows keep their order (ordinals behind a removed row move down).
        Returns the number of rows reclaimed."""
        n = C.c_int64(0)
        check(self._L.krag_index_compact(self._h, C.byref(n)))
        return n.value

    def alive_bitmap(self) -> np.ndarray:
        """the alive bits of the rows (uint32 words, bits past the rows 0)"""
        words = C.c_int64(0)
        check(self._L.krag_index_alive_bitmap(self._h, None, 0, C.byref(words)))
        out = np.zeros(words.value, np.uint32)
        check(self._L.krag_index_alive_bitmap(self._h, ptr(out), out.size, C.byref(words)))
        return out

    # ---- redeal session (kaito_rag.h, krag_redeal_begin): compaction of round-robin shards together, one call per step
    def redeal_begin(self, alive_all: np.ndarray, window_rows: int):
        """alive_all [G, words] uint32 -> (n_windows, n_live, row_bytes, send_rows, send_entries, recv_rows), tables
        [n_windows, G] int64"""
        alive_all = np.ascontiguousarray(alive_all, np.uint32)
        nw, nl, rb = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        check(self._L.krag_redeal_begin(self._h, ptr(alive_all), alive_all.shape[1], window_rows, C.byref(nw), C.byref(nl), C.byref(rb)))
        G = alive_all.shape[0]
        tabs = [np.zeros((nw.value, G), np.int64) for _ in range(3)]
        check(self._L.krag_redeal_tables(self._h, *(ptr(t) for t in tabs)))
        return (nw.value, nl.value, rb.value, *tabs)

    def redeal_prepare(self, recv_entries: np.ndarray):
        recv_entries = np.ascontiguousarray(recv_entries, np.int64)
        check(self._L.krag_redeal_prepare(self._h, ptr(recv_entries)))

    def dev_redeal_pack(self, window: int, d_rows, d_entries, stream=0):
        check(self._L.krag_dev_redeal_pack(self._h, window, ptr(d_rows), ptr(d_entries), ptr(stream)))

    def dev_redeal_unpack(self, window: int, d_rows, d_entries, stream=0):
        check(self._L.krag_dev_redeal_unpack(self._h, window, ptr(d_rows), ptr(d_entries), ptr(stream)))

    def redeal_finish(self, stream=0) -> int:
        n = C.c_int64(0)
        check(self._L.krag_redeal_finish(self._h, ptr(stream), C.byref(n)))
        return n.value

    def redeal_abort(self):
        check(self._L.krag_redeal_abort(self._h))

    def commit(self, vocab: int):
        check(self._L.krag_index_commit(self._h, vocab))

    def commit_local(self, vocab: int):
        df = np.zeros(vocab, np.uint32)
        n_live, total = C.c_int64(0), C.c_int64(0)
        check(self._L.krag_index_commit_local(self._h, vocab, ptr(df), C.byref(n_live), C.byref(total)))
        return df, n_live.value, total.value

    def commit_global(self, vocab: int, df_global, n_docs_global: int, total_len_global: int, ordinal_base: int):
        df_global = np.ascontiguousarray(df_global, np.uint32)
        check(self._L.krag_index_commit_global(self._h, vocab, ptr(df_global), n_docs_global, total_len_global,
                                               ordinal_base))

    def set_ordinal_map(self, base: int, stride: int):
        """global ordinal of local row r = base + r * stride (round-robin shards: base = shard, stride = n_shards)"""
        check(self._L.krag_index_set_ordinal_map(self._h, base, stride))

    def stats(self) -> Stats:
        s = Stats()
        check(self._L.krag_index_stats(self._h, C.byref(s)))
        return s

    def node_ids(self, ordinals) -> np.ndarray:
        ordinals = np.ascontiguousarray(ordinals, np.int64)
        out = np.empty(ordinals.shape, np.uint64)
        check(self._L.krag_index_node_ids(self._h, ordinals.size, ptr(ordinals), ptr(out)))
        return out

    def persist(self, path: str):
        check(self._L.krag_index_persist(self._h, path.encode()))

    def set_dense_mode(self, dense_mode: int, release_shadow: bool = False):
        """KRAG_DENSE_*; DENSE_TC_BF16 builds the bf16 shadow on first use (results stay exact fp32 in every mode)"""
        check(self._L.krag_index_set_dense_mode(self._h, dense_mode, 1 if release_shadow else 0))

    def search_dense(self, q, k: int):
        q = np.ascontiguousarray(q, np.float32).reshape(-1, self.dim)
        b = q.shape[0]
        dist = np.empty((b, k), np.float32)
        ordn = np.empty((b, k), np.int64)
        check(self._L.krag_search_dense(self._h, b, ptr(q), k, ptr(dist), ptr(ordn)))
        return dist, ordn

    @staticmethod
    def _pack_terms(q_terms_list):
        offs = np.zeros(len(q_terms_list) + 1, np.int32)
        for i, t in enumerate(q_terms_list):
            offs[i + 1] = offs[i] + len(t)
        flat = (np.concatenate([np.asarray(t, np.uint32) for t in q_terms_list]) if offs[-1] > 0
                else np.zeros(1, np.uint32))
        return np.ascontiguousarray(flat, np.uint32), offs

    def search_bm25(self, q_terms_list, k: int):
        flat, offs = self._pack_terms(q_terms_list)
        b = len(q_terms_list)
        score = np.empty((b, k), np.float32)
        ordn = np.empty((b, k), np.int64)
        check(self._L.krag_search_bm25(self._h, b, ptr(flat), ptr(offs), k, ptr(score), ptr(ordn)))
        return score, ordn

    def retrieve(self, q, q_terms_list, k: int, cand_mult: float = 3.0, vector_weight: float = 0.7,
                 text_weight: float = 0.3, fusion_mode: int = FUSION_REFERENCE, keyword_allow_bitmap=None):
        """HybridRetriever._aretrieve for a batch. q_terms_list=None -> vector-only fallback."""
        q = np.ascontiguousarray(q, np.float32).reshape(-1, self.dim)
        b = q.shape[0]
        flat = offs = None
        if q_terms_list is not None:
            flat, offs = self._pack_terms(q_terms_list)
        if keyword_allow_bitmap is not None:
            keyword_allow_bitmap = np.ascontiguousarray(keyword_allow_bitmap, np.uint32)
        out = {
            "final": np.empty((b, k), np.float64), "dense": np.empty((b, k), np.float32),
            "sparse": np.empty((b, k), np.float32), "rank": np.empty((b, k), np.int32),
            "ordinal": np.empty((b, k), np.int64), "count": np.empty(b, np.int32),
        }
        check(self._L.krag_retrieve(self._h, b, ptr(q), ptr(flat), ptr(offs), k, cand_mult, vector_weight, text_weight,
                                    fusion_mode, ptr(keyword_allow_bitmap),
                                    0 if keyword_allow_bitmap is None else keyword_allow_bitmap.size, ptr(out["final"]), ptr(out["dense"]),
                                    ptr(out["sparse"]), ptr(out["rank"]), ptr(out["ordinal"]), ptr(out["count"])))
        return out

    # ---- device-pointer stage API ----
    def dev_dense_candidates(self, batch, d_q, P, d_keys, stream=0):
        check(self._L.krag_dev_dense_candidates(self._h, batch, ptr(d_q), P, ptr(d_keys), ptr(stream)))

    def dev_bm25_candidates(self, batch, d_terms, d_toff, P, d_keys, stream=0, h_toff=None):
        """h_toff: optional host copy (int32 [batch+1]) of the offsets; saves a 4-byte device read-back"""
        check(self._L.krag_dev_bm25_candidates(self._h, batch, ptr(d_terms), ptr(d_toff), ptr(h_toff), P, ptr(d_keys),
                                               ptr(stream)))

    # ---- synthetic / inspection ----
    def synth_fill(self, n: int, row_base: int = 0, seed: int = 1, vocab: int = 0):
        check(self._L.krag_synth_fill(self._h, n, row_base, seed, vocab))

    def read_rows(self, row0: int, n: int) -> np.ndarray:
        out = np.empty((n, self.dim), np.float32)
        check(self._L.krag_index_read_rows(self._h, row0, n, ptr(out)))
        return out

    def debug_tc_dump(self, q) -> np.ndarray:
        """K2 raw output a[j, r] = |x_r|^2 - 2 x_r.q_j for all rows (test hook)."""
        q = np.ascontiguousarray(q, np.float32).reshape(-1, self.dim)
        S, nqp = C.c_int64(0), C.c_int32(0)
        check(self._L.krag_debug_tc_dump(self._h, q.shape[0], ptr(q), None, 0, C.byref(S), C.byref(nqp)))
        out = np.empty((nqp.value, S.value), np.float32)
        check(self._L.krag_debug_tc_dump(self._h, q.shape[0], ptr(q), ptr(out), out.size, C.byref(S), C.byref(nqp)))
        return out

    def debug_tc_dump_pass(self, q, tc_pass: int) -> np.ndarray:
        """a[j, r] = |x_r|^2 - 2 x_r.q_j from one prune pass (TC_PASS_*) over every row: [nq_pad, S] (test hook)"""
        q = np.ascontiguousarray(q, np.float32).reshape(-1, self.dim)
        S, nqp = C.c_int64(0), C.c_int32(0)
        check(self._L.krag_debug_tc_dump_pass(self._h, tc_pass, q.shape[0], ptr(q), None, 0, C.byref(S), C.byref(nqp)))
        out = np.empty((nqp.value, S.value), np.float32)
        check(self._L.krag_debug_tc_dump_pass(self._h, tc_pass, q.shape[0], ptr(q), ptr(out), out.size, C.byref(S), C.byref(nqp)))
        return out

    def debug_tc_prune(self, q, thr, cap: int, tc_pass: int):
        """one main prune pass (TC_PASS_*) with thresholds thr [nq_pad] (nq_pad = 64, 128 or 256, the NQ bucket of the
        batch): (counts uint32 [nq_pad], rows uint32 [nq_pad, cap], valid in each row up to min(count, cap)) (test hook)"""
        q = np.ascontiguousarray(q, np.float32).reshape(-1, self.dim)
        nqp = 64 if q.shape[0] <= 64 else (128 if q.shape[0] <= 128 else 256)
        thr = np.ascontiguousarray(thr, np.float32)
        if thr.shape != (nqp,):
            raise ValueError(f"thr must hold {nqp} thresholds, one per query column of the NQ bucket")
        counts = np.zeros(nqp, np.uint32)
        rows = np.zeros((nqp, cap), np.uint32)
        check(self._L.krag_debug_tc_prune(self._h, tc_pass, q.shape[0], ptr(q), ptr(thr), cap, ptr(counts), ptr(rows)))
        return counts, rows

    def debug_stored_rows(self, row0: int, n: int) -> np.ndarray:
        """rows [row0, row0 + n) as the device stores them: uint32 [n, dim_padded] (test hook)"""
        out = np.empty((n, self.stats().dim_padded), np.uint32)
        check(self._L.krag_debug_read_stored_rows(self._h, row0, n, ptr(out)))
        return out

    def read_postings(self, term: int, cap: int = 1 << 22):
        cnt = C.c_int64(0)
        docs = np.empty(cap, np.uint32)
        scores = np.empty(cap, np.float32)
        check(self._L.krag_index_read_postings(self._h, term, cap, ptr(docs), ptr(scores), C.byref(cnt)))
        m = min(cnt.value, cap)
        return docs[:m], scores[:m], cnt.value
