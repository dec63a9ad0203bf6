/*
 * kaito_rag.h -- C ABI of libkaito_rag.so, the H100 (sm_90a) retrieval engine behind
 * KAITO's RAGService /retrieve and /index.
 *
 * The reference has no in-process FFI seam: its service is Python calling pip wheels
 * (faiss-cpu, bm25s) -- SURVEY.md section 8(b).  This header is the seam a Go (cgo) or
 * Python (ctypes) RAGService host binds instead of those wheels.  Each entry point
 * names the reference call it replaces (paths relative to presets/ragengine/).
 *
 * Conventions
 *   - every call returns int32 status: 0 = KRAG_OK, negative = KRAG_E_*;
 *     krag_last_error() returns a thread-local UTF-8 message for the last failure.
 *   - caller owns host buffers; the library owns device memory; handles are opaque.
 *   - NO CPU FALLBACK: without an sm_90 device krag_init fails with KRAG_E_NO_DEVICE.
 *   - thread-safety mirrors the reference's aiorwlock (vector_store/base.py:77-79):
 *     searches on one index may run concurrently, mutations are exclusive.
 *   - "ordinal" = position of a node in insertion order (global across shards:
 *     shard base + local row).  Ties everywhere break by ascending ordinal.
 *   - candidate keys are u64: high 32 bits = order-preserving bits of the fp32 value
 *     (dense: L2^2 ascending; bm25: complemented, so ascending key == descending
 *     score), low 32 bits = global ordinal.  KRAG_KEY_PAD (all ones) pads short lists.
 */
#ifndef KAITO_RAG_H_
#define KAITO_RAG_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KRAG_OK 0
#define KRAG_E_INVALID (-1)     /* bad argument */
#define KRAG_E_NO_DEVICE (-2)   /* no sm_90 CUDA device / driver */
#define KRAG_E_CUDA (-3)        /* CUDA runtime error (message has details) */
#define KRAG_E_OOM (-4)         /* device or host allocation failed */
#define KRAG_E_NOT_FOUND (-5)   /* unknown index / node id */
#define KRAG_E_STATE (-6)       /* call not valid in the current state (e.g. search before commit) */
#define KRAG_E_IO (-7)          /* persist / load failure */
#define KRAG_E_UNSUPPORTED (-8) /* feature compiled out or not available on this device */

#define KRAG_KEY_PAD 0xFFFFFFFFFFFFFFFFull
#define KRAG_MAX_TOP_K 300   /* config.py:127 RAG_MAX_TOP_K */
#define KRAG_MAX_POOL 1024   /* >= int(300 * 3.0) = 900, hybrid_retriever.py:97-98 */

#define KRAG_FUSION_REFERENCE 0  /* vec_score = L2^2 itself (hybrid_retriever.py:139-142,158-166) */
#define KRAG_FUSION_SIMILARITY 1 /* vec_score = 1 - L2^2/2 (not the reference) */
/* OR-ed into fusion_mode: apply krag_retrieve's allow bitmap INSIDE the dense and BM25 kernels (every one of the P
 * candidates of both lists satisfies the filter) instead of the reference's post-filter of the keyword list only
 * (hybrid_retriever.py:227-235; its dense side cannot filter at all, SURVEY.md section 8 a9).  Not the reference. */
#define KRAG_FILTER_PUSHDOWN 0x100

#define KRAG_DENSE_AUTO 0   /* exact fp32 scan for small batches, tensor-core path for large */
#define KRAG_DENSE_SCAN 1   /* K1: exact fp32 CUDA-core scan */
#define KRAG_DENSE_TC 2     /* K2: wgmma prune pass (bf16 wgmma on the bf16 high halves the device rows are stored with;
                               TF32 when the padded dimension is not a multiple of 64) + exact fp32 rescoring */
#define KRAG_DENSE_TC_BF16 3 /* K2 pruning on a bf16 SHADOW copy of the corpus (+50% memory); the returned distances are
                               still exact fp32 re-scores of the fp32 corpus and carry the same exactness certificate */

#define KRAG_DENSE_TC_TF32 4 /* K2 with the fp32 rows consumed directly as TF32 (tf32 wgmma), kept for comparison */

/* Where an index keeps its fp32 rows (krag_config.row_storage; every index created or loaded in the context).
 * HOST: the fp32 rows live in pinned host memory; the device holds a bf16 copy (2 B per element) plus 8 B per row of
 * metadata.  Searches prune on the bf16 copy and rescore exactly from the host rows: returned distances and ids are
 * bit-identical to DEVICE mode, ties included.  KRAG_DENSE_SCAN streams the host rows through the exact scan instead. */
#define KRAG_ROWS_DEVICE 0
#define KRAG_ROWS_HOST 1

typedef struct krag_ctx krag_ctx;
typedef struct krag_index krag_index;

typedef struct krag_config {
    int32_t device_id;      /* CUDA device ordinal */
    int32_t rank;           /* shard rank of this process (0 when single GPU) */
    int32_t world_size;     /* number of shards (1 when single GPU) */
    int32_t dense_mode;     /* KRAG_DENSE_* */
    int32_t search_slots;   /* concurrent search workspaces (0 = default 4) */
    int32_t row_storage;    /* KRAG_ROWS_* (0 = device) */
    int32_t reserved[2];
} krag_config;

typedef struct krag_stats_t {
    int64_t n_rows;         /* local dense rows (incl. tombstoned) */
    int64_t n_live;         /* local live rows */
    int64_t nnz;            /* local postings */
    int64_t n_docs_global;  /* BM25 N used for idf */
    int64_t total_len_global;
    int64_t vocab;
    int64_t ordinal_base;   /* global ordinal of local row 0 */
    int32_t dim;            /* logical dimension */
    int32_t dim_padded;     /* row stride in floats (multiple of 32) */
    int32_t committed;      /* postings valid for the current rows */
    int32_t reserved;
    int64_t device_bytes;   /* device memory held by this index */
} krag_stats_t;

/* --------------------------------------------------------------------- lifecycle */
int32_t krag_version(void);
const char* krag_last_error(void);
/* replaces: process-wide FAISS/BM25 imports of the RAGService (main.py:141-158) */
int32_t krag_init(const krag_config* cfg, krag_ctx** out);
int32_t krag_shutdown(krag_ctx* ctx);
/* number of kernels this library has launched since krag_init (bench.py gpu_launches) */
int64_t krag_launch_count(krag_ctx* ctx);
/* device memory this process currently holds through libkaito_rag, in bytes (every context, index and embedder) */
int64_t krag_device_bytes(void);
/* pinned host memory this process currently holds through libkaito_rag, in bytes (KRAG_ROWS_HOST rows) */
int64_t krag_host_pinned_bytes(void);
void* krag_ctx_stream(krag_ctx* ctx);  /* cudaStream_t of search slot 0 (for event timing) */

/* ------------------------------------------------------------------------- index */
/* replaces: faiss.IndexIDMap(faiss.IndexFlatL2(dim)) + FaissMapVectorStore,
 * vector_store/faiss_store.py:41-50 */
int32_t krag_index_create(krag_ctx* ctx, const char* name, int32_t dim, krag_index** out);
/* replaces: BaseVectorStore.delete_index (DELETE /indexes/{name}, main.py:774) */
int32_t krag_index_drop(krag_index* idx);
int32_t krag_index_reserve(krag_index* idx, int64_t rows, int64_t nnz);
/*
 * Append n nodes.  replaces: FaissMapVectorStore.add -> index.add_with_ids and the
 * docstore insert that BM25Retriever.from_defaults later tokenises
 * (vector_store/base.py:155-166, :499-511; hybrid_retriever.py:122-125).
 *   node_ids     [n]            caller-chosen unique u64 handles
 *   vecs         [n, dim]       fp32 row-major embeddings
 *   term_offsets [n+1]          CSR offsets into term_ids/term_tf (NULL: no sparse side)
 *   term_ids     [nnz]          unique term ids per node (host vocabulary)
 *   term_tf      [nnz]          term frequency within the node
 *   doc_len      [n]            token count of the node after stop-word removal
 */
int32_t krag_index_add(krag_index* idx, int64_t n, const uint64_t* node_ids, const float* vecs,
                       const int64_t* term_offsets, const uint32_t* term_ids, const uint16_t* term_tf,
                       const uint32_t* doc_len);
/* replaces: IndexIDMap.remove_ids via llama-index delete (vector_store/base.py:563-643) */
int32_t krag_index_remove(krag_index* idx, int64_t n, const uint64_t* node_ids, int64_t* n_removed);
/* Remove tombstoned rows from the index: live rows keep their relative order and move down to rows [0, n_live).
 * Node ids, vectors, term lists, BM25 scores and every search result (ids, scores, tie order) are unchanged; only the
 * ordinals of rows behind a removed row change.  Takes the index's writer lock.  *n_reclaimed_out = rows removed.
 * The rows move in place on the device (a bounded staging buffer, no second copy of the index); the committed postings
 * are renumbered with the scores of the last commit (an uncommitted index stays uncommitted and keeps them for its next commit).  Buffers that shrank
 * are reallocated at their exact size when that fits beside the old ones.  No dead rows: a no-op, 0 reclaimed.
 * KRAG_E_UNSUPPORTED for an ordinal stride > 1 (round-robin shards, krag_index_set_ordinal_map): the index is unchanged.
 * No counterpart in the reference, whose FAISS IndexIDMap.remove_ids compacts on every delete. */
int32_t krag_index_compact(krag_index* idx, int64_t* n_reclaimed_out);
/* Copy of the alive bitmap (bit r of word r / 32 = local row r is live; bits past the rows are 0).  *words_out =
 * (n_rows + 31) / 32; out == NULL only reports it.  The input of krag_redeal_begin. */
int32_t krag_index_alive_bitmap(krag_index* idx, uint32_t* out, int64_t cap_words, int64_t* words_out);
/*
 * Redeal: compaction of the G round-robin shards of one index together (shard s = ordinal map (s, G), one per rank; no
 * counterpart in the reference).  Afterwards shard s, row j holds the live row whose new global ordinal is j * G + s: the
 * layout a fresh service builds by inserting only the live nodes, in their old order.  Node ids become the new ordinals
 * (every node id must equal its ordinal before).  Vectors, the bf16 copy, norms, doc lengths and term lists move; the
 * postings are dropped, so the session ends with the collective commit (commit_local -> all-reduce -> commit_global), a
 * full build under the last commit's statistics.  Rows move between ranks in windows of new ordinals over a transport the
 * host provides (kaito_b200/sharded.py: all_to_all_single).  Every rank, in the same order:
 *   1. krag_index_alive_bitmap; the host gathers every shard's bitmap, padded to the longest: alive_all [G][words].
 *   2. krag_redeal_begin: the plan.  KRAG_E_STATE when rows were added or removed since the last commit, or a node id
 *      differs from its ordinal.  n_windows, n_live (over all shards) and row_bytes (payload of one row) come back.
 *   3. krag_redeal_tables: [n_windows][G] rows and term entries this shard sends to each shard, rows it receives from each.
 *      The host exchanges the entry tables: recv_entries[k][t] = send_entries of shard t for window k, this shard.
 *   4. krag_redeal_prepare(recv_entries): allocates the new term arrays.  Until here nothing has changed: on any failure
 *      krag_redeal_abort on every rank leaves every shard as it was.
 *   5. per window k = 0 .. n_windows-1: krag_dev_redeal_pack (this shard's rows of the window into d_rows, row_bytes
 *      each, and their entries into d_entries, 8 B each, grouped by destination shard), the exchange of both buffers
 *      (split sizes from the tables), krag_dev_redeal_unpack (the received buffers, grouped by source shard).  Device
 *      pointers, ordered on `stream` (cudaStream_t).
 *   6. krag_redeal_finish: *n_rows_out = this shard's rows; then the collective commit.
 * While a session is open every other call on the index returns KRAG_E_STATE.  After the first unpack the rows are in
 * flight: a failure (or krag_redeal_abort) from there on leaves the index unusable and only krag_index_drop is allowed.
 * krag_last_compact reports the session: move_ms from the first pack to the finish, postings_ms 0, rows_moved and
 * bytes_moved = what this shard sent.  window_rows bounds the rows of one window (staging: up to window_rows rows sent and
 * window_rows / G + 1 received per window).
 */
int32_t krag_redeal_begin(krag_index* idx, const uint32_t* alive_all /*[G][words] host*/, int64_t words, int64_t window_rows,
                          int64_t* n_windows_out, int64_t* n_live_out, int64_t* row_bytes_out);
int32_t krag_redeal_tables(krag_index* idx, int64_t* send_rows, int64_t* send_entries, int64_t* recv_rows /*[n_windows][G] each*/);
int32_t krag_redeal_prepare(krag_index* idx, const int64_t* recv_entries /*[n_windows][G]*/);
int32_t krag_dev_redeal_pack(krag_index* idx, int64_t window, void* d_rows, void* d_entries, void* stream);
int32_t krag_dev_redeal_unpack(krag_index* idx, int64_t window, const void* d_rows, const void* d_entries, void* stream);
int32_t krag_redeal_finish(krag_index* idx, void* stream, int64_t* n_rows_out);
int32_t krag_redeal_abort(krag_index* idx);
/*
 * (Re)build BM25 postings for the rows added so far.  replaces the per-query
 * BM25Retriever.from_defaults rebuild (hybrid_retriever.py:104-130): same scores,
 * built once.  After the first commit, a commit merges the added and removed rows into the
 * committed postings on the device (bit-identical to a full build; krag_last_commit).  Single-shard form:
 */
int32_t krag_index_commit(krag_index* idx, int64_t vocab);
/* Multi-shard form: each rank reports local stats, the host all-reduces them (sum),
 * then every rank finishes with the global values (SURVEY.md section 8e). */
int32_t krag_index_commit_local(krag_index* idx, int64_t vocab, uint32_t* df_out /*[vocab] host*/,
                                int64_t* n_live_out, int64_t* total_len_out);
int32_t krag_index_commit_global(krag_index* idx, int64_t vocab, const uint32_t* df_global /*[vocab] host*/,
                                 int64_t n_docs_global, int64_t total_len_global, int64_t ordinal_base);
/* Global ordinal of local row r = ordinal_base + r * ordinal_stride (default base 0 / stride 1; krag_index_commit_global sets
 * the base of a contiguous shard).  The multi-GPU service deals nodes round-robin over G shards (node o -> shard o % G, row
 * o / G) and sets (base, stride) = (shard, G): ordinals -- and with them every tie-break -- equal the single-GPU insertion
 * order.  Call before krag_index_commit_global / searches; no counterpart in the reference (one replica, manifests.go:81). */
int32_t krag_index_set_ordinal_map(krag_index* idx, int64_t ordinal_base, int64_t ordinal_stride);
int32_t krag_index_stats(krag_index* idx, krag_stats_t* out);
/* ordinals (global) -> node ids for rows of THIS shard; KRAG_E_NOT_FOUND if out of range */
int32_t krag_index_node_ids(krag_index* idx, int64_t n, const int64_t* ordinals, uint64_t* node_ids_out);
/* replaces: StorageContext.persist / load_index_from_storage (vector_store/base.py:779-868) */
int32_t krag_index_persist(krag_index* idx, const char* dir);
int32_t krag_index_load(krag_ctx* ctx, const char* name, const char* dir, krag_index** out);

/* ------------------------------------------------- search, host buffers (1 shard) */
/*
 * replaces: IndexIDMap(IndexFlatL2).search(q, k) reached from
 * index.as_retriever(similarity_top_k=P).aretrieve (hybrid_retriever.py:209-213).
 *   q [batch, dim] fp32;  out_l2sq [batch, k] ascending (+inf pad);
 *   out_ordinals [batch, k] (-1 pad, like faiss' -1 labels).
 */
int32_t krag_search_dense(krag_index* idx, int32_t batch, const float* q, int32_t k,
                          float* out_l2sq, int64_t* out_ordinals);
/*
 * replaces: bm25_retriever.aretrieve(query) (hybrid_retriever.py:220) after host-side
 * tokenisation.  q_terms are term ids in query order, duplicates kept;
 * q_term_offsets [batch+1].  out_score [batch,k] descending; zero-score documents fill
 * short lists as bm25s' argpartition does; out_ordinals -1 past the live doc count.
 */
int32_t krag_search_bm25(krag_index* idx, int32_t batch, const uint32_t* q_terms, const int32_t* q_term_offsets,
                         int32_t k, float* out_score, int64_t* out_ordinals);
/*
 * The whole HybridRetriever._aretrieve (hybrid_retriever.py:205-237) for a batch:
 * dense top-P, BM25 top-P, keyword-side metadata post-filter (optional bitmap of
 * allowed LOCAL rows, 1 bit per row, at least (n_rows + 31) / 32 words -- fewer is KRAG_E_INVALID; NULL = no filter),
 * _fuse, top-k.
 *   P = int(k * max(1, cand_mult)).  q_terms == NULL or an uncommitted index selects
 *   the reference's vector-only fallback (:216-218): dense top-P cut to k.
 * Outputs are [batch, k]; out_count[batch] gives the valid prefix per query.
 *   out_final  fp64 fused score (dense-only fallback: the L2^2)
 *   out_dense  L2^2 or NaN;  out_sparse BM25 score or NaN;  out_rank BM25 rank or -1
 * fusion_mode | KRAG_FILTER_PUSHDOWN: the bitmap restricts both candidate scans instead (also in the vector-only case).
 */
int32_t krag_retrieve(krag_index* idx, int32_t batch, const float* q,
                      const uint32_t* q_terms, const int32_t* q_term_offsets,
                      int32_t k, double cand_mult, double vector_weight, double text_weight, int32_t fusion_mode,
                      const uint32_t* keyword_allow_bitmap, int64_t keyword_allow_words /* u32 words held by the bitmap */,
                      double* out_final, float* out_dense, float* out_sparse, int32_t* out_rank,
                      int64_t* out_ordinals, int32_t* out_count);

/* ------------------------------- stage API, DEVICE pointers (one process per GPU) */
/* All pointers are device pointers valid on ctx's device; `stream` is a cudaStream_t
 * (NULL = legacy default stream).  These let the host place one NCCL all-gather
 * between the local candidate stage and the merge/fuse stage (SURVEY.md section 8e).
 * The candidate stages return with their work still queued on `stream`.  That work is
 * ordered before every later search that reuses its workspace (search_slots of them per
 * context) and before every later mutation of the index: a mutation first waits for it
 * (the host blocks until it has finished), so queued kernels never see rows, tombstones
 * or postings change under them. */
int32_t krag_dev_dense_candidates(krag_index* idx, int32_t batch, const float* d_q, int32_t P,
                                  uint64_t* d_keys_out /*[batch,P]*/, void* stream);
int32_t krag_dev_bm25_candidates(krag_index* idx, int32_t batch, const uint32_t* d_q_terms,
                                 const int32_t* d_q_term_offsets, const int32_t* h_q_term_offsets,
                                 int32_t P, uint64_t* d_keys_out /*[batch,P]*/, void* stream);
/* keys_in [n_lists, batch, P] -> keys_out [batch, P]: the P smallest keys per query */
int32_t krag_dev_merge(krag_ctx* ctx, int32_t n_lists, int32_t batch, int32_t P, const uint64_t* d_keys_in,
                       uint64_t* d_keys_out, void* stream);
/* HybridRetriever._fuse (hybrid_retriever.py:132-166) on merged candidate lists.
 * d_bm25_keys == NULL selects the vector-only fallback. d_allow: optional bitmap over
 * GLOBAL ordinals for the keyword-side post-filter (:227-235). */
int32_t krag_dev_fuse(krag_ctx* ctx, int32_t batch, int32_t P, int32_t k, const uint64_t* d_dense_keys,
                      const uint64_t* d_bm25_keys, double vector_weight, double text_weight, int32_t fusion_mode,
                      const uint32_t* d_allow, double* d_out_final, float* d_out_dense, float* d_out_sparse,
                      int32_t* d_out_rank, int64_t* d_out_ordinals, int32_t* d_out_count, void* stream);

/* ------------------------------------------------ synthetic corpora (bench / tests) */
/* Fill the index with n deterministic unit-norm rows generated ON THE DEVICE
 * (counter-based Philox4x32-10 keyed by seed and global row), plus, when vocab > 0,
 * Zipf(s=1.07) term lists with log-normal lengths (SURVEY.md section 8d).  Node id of a
 * synthetic row == its global ordinal.  Not on the product path. */
int32_t krag_synth_fill(krag_index* idx, int64_t n, int64_t row_base, uint64_t seed, int64_t vocab);
/* copy rows [row0,row0+n) back to host (parity spot checks at full size) */
int32_t krag_index_read_rows(krag_index* idx, int64_t row0, int64_t n, float* out /*[n,dim]*/);
/* copy the postings of one term back to host: returns count via *n_out (cap entries max) */
int32_t krag_index_read_postings(krag_index* idx, uint32_t term, int64_t cap, uint32_t* docs_out, float* scores_out,
                                 int64_t* n_out);

/* ----------------------------------------- peer-memory candidate exchange (one process per GPU, one box) */
/* The all-gather + merge of the per-shard candidate lists done by our own kernels over NVLink peer memory:
 * every rank creates a mailbox (cudaMalloc + CUDA IPC handle), the host exchanges the 64-byte handles (any
 * side channel; kaito_b200/sharded.py uses torch.distributed.all_gather_object), every rank connects, and
 * krag_dev_exchange_merge then (1) stores this rank's lists [n_lists, batch, P] into all mailboxes with P2P
 * writes + a system-scope release flag and (2) waits for all ranks' flags and merges G*P -> P locally.
 * No counterpart in the reference (single replica, SURVEY.md section 8e). */
typedef struct krag_p2p krag_p2p;
int32_t krag_p2p_create(krag_ctx* ctx, int32_t rank, int32_t world, int32_t max_batch, int32_t max_P, krag_p2p** out,
                        uint8_t* handle_out /*[64]*/);
int32_t krag_p2p_connect(krag_p2p* p, const uint8_t* handles /*[world][64], own entry ignored*/);
int32_t krag_dev_exchange_merge(krag_p2p* p, int32_t n_lists, int32_t batch, int32_t P, const uint64_t* d_local_keys,
                                uint64_t* d_merged_out /*[n_lists, batch, P]*/, void* stream);
int32_t krag_p2p_destroy(krag_p2p* p);

/* ------------------------------------------------------------- embedding forward (K5) */
/* replaces: LocalHuggingFaceEmbedding (embedding/huggingface_local_embedding.py:34-53) -> sentence-
 * transformers BertModel forward, CLS or mean pooling, L2 normalisation.  Tokenisation (WordPiece) stays in
 * the host.  Weights are loaded by their Hugging Face BertModel names ("embeddings.word_embeddings.weight",
 * "encoder.layer.0.attention.self.query.weight", ...), fp32, row-major as torch stores them.
 * MPNet (all-mpnet-base-v2, multi-qa-mpnet-*): an embedder loaded with "encoder.relative_attention_bias.weight"
 * [32 buckets, heads] (transformers MPNetModel's name) is an MPNet encoder: every attention score of head h gets
 * weight[bucket][h], bucket = MPNetEncoder.relative_position_bucket(key - query, 32 buckets, max distance 128) (see
 * krag_debug_relative_bucket).  The host loads the other MPNet tensors under the BERT names (attention.attn.q -> .self.query,
 * .k -> .self.key, .v -> .self.value, .o -> .output.dense, attention.LayerNorm -> attention.output.LayerNorm), a zero
 * token-type table with type_vocab = 1, and sets the position offset to 2.  finalize: KRAG_E_INVALID, naming the tensor,
 * when it does not hold 32 * heads elements.
 * nomic-bert (nomic-embed-text-v1 / -v1.5) is a post-LN BERT with two variants, each selectable alone:
 *  - rotary positions (krag_embedder_set_rotary with base > 0, before finalize): no position table is read (none need be
 *    loaded); Q and K of token i of a sequence (position off + i) are rotated as transformers' default RoPE does,
 *    q' = q cos + rotate_half(q) sin, pairing element j < dh/2 of a head with j + dh/2, at the fp32 angle fp32(pos) *
 *    (1 / base^(2j / dh)) (see krag_debug_rotary_cos_sin).  Sequences may hold max_position - off tokens.
 *  - a gated FFN (SwiGLU): an embedder loaded with "encoder.layer.{l}.intermediate.gate.weight" [intermediate, hidden] and
 *    "encoder.layer.{l}.intermediate.gate.bias" [intermediate] computes output.dense(silu(gate . h) * (intermediate.dense . h))
 *    in place of output.dense(gelu(intermediate.dense . h)); intermediate.dense is the up projection.
 * nomic has no Linear biases: the host loads zero biases under every BERT bias name (and the gate's), a zero token-type row
 * if the checkpoint has none, and maps the names (see INTEGRATION.md).  finalize: KRAG_E_INVALID, naming the tensor, when a
 * gate tensor has the wrong size or is loaded on some layers but not others, or when rotary is off and the position table
 * is missing. */
typedef struct krag_embedder krag_embedder;
typedef struct krag_bert_config {
    int32_t layers, hidden, heads, intermediate, vocab, max_position, type_vocab;
    float ln_eps;
} krag_bert_config;
int32_t krag_embedder_create(krag_ctx* ctx, const krag_bert_config* cfg, krag_embedder** out);
int32_t krag_embedder_load_tensor(krag_embedder* e, const char* name, const float* data, int64_t n_elems);
/* KRAG_E_INVALID, naming the tensor, when one is missing or its element count is not the config's (word table
 * vocab * hidden, position table max_position * hidden, token-type table type_vocab * hidden, ...) */
int32_t krag_embedder_finalize(krag_embedder* e);
/* tok_ids: packed token ids of all sequences ([CLS] ... [SEP] each); tok_offsets [batch+1]; out [batch, hidden] */
int32_t krag_embed(krag_embedder* e, int32_t batch, const int32_t* tok_ids, const int32_t* tok_offsets, float* out);
/* same, result left on the device: rows of d_out with stride ld_out floats (>= hidden; the padded query layout
 * krag_dev_dense_candidates takes); `stream` (cudaStream_t) is made to wait for the embeddings. tok_* are HOST. */
int32_t krag_embed_dev(krag_embedder* e, int32_t batch, const int32_t* tok_ids, const int32_t* tok_offsets, float* d_out,
                       int32_t ld_out, void* stream);
/* Pooling of the last hidden state before the L2 normalisation (sentence-transformers' Pooling module, read from the
 * snapshot's modules.json and <pooling dir>/config.json by the host): the [CLS] row (default), or the mean over every token
 * of the sequence, [CLS] and [SEP] included.  May be called before or after finalize and between forwards; any other
 * mode is KRAG_E_INVALID. */
#define KRAG_POOL_CLS 0
#define KRAG_POOL_MEAN 1
int32_t krag_embedder_set_pooling(krag_embedder* e, int32_t mode);
/* Arithmetic of the encoder's GEMM and attention products, for every forward of this embedder (krag_embed, krag_embed_dev,
 * krag_rerank).  KRAG_PRECISION_FP32 (default): split-fp16 operands, three tensor-core products per step, results held to
 * fp32 arithmetic.  KRAG_PRECISION_FP16: operands rounded to fp16 (round to nearest even, saturating at the largest finite
 * value), one tensor-core product per step with fp32 accumulation; bias, GELU, the residual stream, LayerNorm, softmax and the
 * classifier head stay fp32.  Meant for cross-encoder scores, which are only compared with each other.  Embeddings computed in
 * fp16 mode are OUTSIDE the 1e-4 score contract of the dense search: a host that stores or queries with them does so
 * knowingly.  The weights are shared by both modes (no second copy).  May be called before or after finalize and between
 * forwards; any other mode is KRAG_E_INVALID. */
#define KRAG_PRECISION_FP32 0
#define KRAG_PRECISION_FP16 1
int32_t krag_embedder_set_precision(krag_embedder* e, int32_t mode);
/* Position row of a sequence's first token (default 0): token i of every sequence takes position row off + i, so a
 * sequence may hold at most max_position - off tokens (else the forward is KRAG_E_INVALID).  RoBERTa / XLM-RoBERTa models
 * number positions from pad_token_id + 1 (= 2).  off >= 0; may be called before or after finalize and between forwards. */
int32_t krag_embedder_set_position_offset(krag_embedder* e, int32_t off);
/* Under CLS pooling the last layer's O projection, FFN and LayerNorms run on the [CLS] rows only (on = 1, the default).
 * on = 0 runs them over every token; the embeddings are the same bits either way.  Test hook. */
int32_t krag_debug_embedder_cls_rows(krag_embedder* e, int32_t on);
/* The relative-position bucket an MPNet embedder's attention applies at rel = key position - query position: transformers'
 * MPNetEncoder.relative_position_bucket with 32 buckets and max distance 128 (the distance is clamped to [-128, 128] first,
 * which changes no bucket).  Host-only: needs no device.  Test hook. */
int32_t krag_debug_relative_bucket(int32_t rel);
/* Rotary positions (nomic-bert): base = the model's rotary base (rotary_emb_base / rope_theta; nomic: 1000), 0 = off (the
 * default: the position table).  Takes effect at the next krag_embedder_finalize.  base < 0 or infinite: KRAG_E_INVALID. */
int32_t krag_embedder_set_rotary(krag_embedder* e, float base);
/* The fp32 cos and sin a rotary embedder applies at position pos to pairs j = 0 .. dh/2 - 1 of a head (cos_out, sin_out:
 * dh/2 floats each): the angle fp32(pos) * inv_freq[j], inv_freq[j] = 1 / base^(2j / dh), both fp32 as torch computes
 * them.  Host-only: needs no device.  Test hook. */
int32_t krag_debug_rotary_cos_sin(float base, int32_t dh, int32_t pos, float* cos_out, float* sin_out);
/* Cross-encoder reranking (BertForSequenceClassification with one label).  The embedder must have been loaded with the
 * head as well: "pooler.dense.weight" [hidden, hidden], "pooler.dense.bias", "classifier.weight" [1, hidden] and
 * "classifier.bias" [1].  Query i owns pairs pair_offsets[i] .. pair_offsets[i+1] (0 to 300 of them); pair p is the packed
 * sequence tok_ids[tok_offsets[p] .. tok_offsets[p+1]) = [CLS] query [SEP] passage [SEP] (at most max_position - the
 * position offset tokens), whose tokens from seg_b[p] on (the first passage token, in [1, length]) take token type 1.
 * seg_b = NULL: unsegmented pairs, every token takes token type 0 (XLM-RoBERTa's <s> query </s></s> passage </s>; any
 * type_vocab >= 1).  score = activation(classifier . tanh(pooler([CLS] row))); an XLM-RoBERTa head (classifier.dense,
 * classifier.out_proj) is the same arithmetic, loaded under the pooler / classifier names.  out_pos / out_score [n_queries, top_k]: per query its best top_k pairs (position within the
 * query's pairs), scores descending, equal scores by position ascending; -1 / NaN past the query's pair count.  All
 * arguments are HOST memory; the call returns synchronised.  KRAG_E_INVALID: head missing, top_k outside [1, 300],
 * unknown activation, a pair too long or seg_b out of range. */
#define KRAG_RERANK_SIGMOID 0
#define KRAG_RERANK_IDENTITY 1
int32_t krag_rerank(krag_embedder* e, int32_t n_queries, const int32_t* pair_offsets, const int32_t* tok_ids,
                    const int32_t* tok_offsets, const int32_t* seg_b, int32_t activation, int32_t top_k, int32_t* out_pos,
                    float* out_score);
/* Late-interaction reranking (ColBERT: colbertv2.0, answerai-colbert-small).  krag_embedder_set_late_interaction, before
 * krag_embedder_finalize: the projection linear.weight [dim, hidden] (no bias; dim a multiple of 16 in [16, 256]).
 * KRAG_E_INVALID, naming linear.weight, when n_elems is not dim * hidden.  Every token row of the last layer then maps to
 * v = W h / max(|W h|, 1e-12); the forward gives each sequence bits that depend on its own tokens alone (no split-K GEMM
 * plan, the 64-key attention blocking at every length). */
int32_t krag_embedder_set_late_interaction(krag_embedder* e, int32_t dim, const float* weight, int64_t n_elems);
/* Query i is query_tok[i * query_len .. (i+1) * query_len) (query_len <= 32; ColBERT's [CLS] [Q] q... [SEP] [MASK]...) whose
 * keys are its first query_keys[i] rows (1 .. query_len; every row is a query and an output row).  Passage p is
 * passage_tok[passage_offsets[p] .. passage_offsets[p+1]); row t enters the max iff passage_keep[t] != 0 (at least one row
 * of every passage must).  Query i owns pairs pair_offsets[i] .. pair_offsets[i+1] (0 to 300), pair j scores passage
 * pair_passage[j]: score = sum over the query's rows r, in order, of the max over kept passage rows of the fp32 dot product
 * of their unit vectors.  Each query and passage is encoded once per call, however many pairs name it.  out_pos /
 * out_score [n_queries, top_k] as for krag_rerank.  All arguments are HOST memory; the call returns synchronised. */
int32_t krag_late_rerank(krag_embedder* e, int32_t n_queries, int32_t query_len, const int32_t* query_tok, const int32_t* query_keys,
                         int32_t n_passages, const int32_t* passage_tok, const int32_t* passage_offsets, const uint8_t* passage_keep,
                         const int32_t* pair_offsets, const int32_t* pair_passage, int32_t top_k, int32_t* out_pos, float* out_score);
/* The unit token vectors [tok_offsets[batch], dim] of packed sequences (key_lens [batch] or NULL: every row a key), as
 * krag_late_rerank computes them.  Test hook. */
int32_t krag_debug_late_vectors(krag_embedder* e, int32_t batch, const int32_t* tok_ids, const int32_t* tok_offsets, const int32_t* key_lens,
                                float* out);
/* Passage vector stores.  A store keeps, per ordinal, a passage's kept unit vectors (the rows krag_late_rerank lets into the
 * max, in row order, fp32 [rows, dim]) in device slabs of at most 256 MB; they have the bits krag_debug_late_vectors gives
 * for that passage alone, so a pair scored from a stored passage has the score it has when the passage is encoded in the
 * call.  Every store created from one embedder draws its slabs from one budget of device bytes
 * (krag_embedder_set_store_budget, default 0: nothing is stored; KRAG_E_INVALID when negative).  A store records the
 * embedder's precision mode; an append or rerank under another mode is KRAG_E_INVALID.  The embedder cannot be destroyed
 * while it has stores (KRAG_E_INVALID). */
typedef struct krag_late_store krag_late_store;
int32_t krag_embedder_set_store_budget(krag_embedder* e, int64_t bytes);
int32_t krag_late_store_create(krag_embedder* e, krag_late_store** out);
int32_t krag_late_store_destroy(krag_late_store* s);
/* Passages p < n (passage_tok / passage_offsets / passage_keep as for krag_late_rerank, with its checks) become the next n
 * ordinals, in order.  stored_out [n]: 1 where the passage was stored, 0 where the budget (or the device) had no room; an
 * unstored ordinal is then scored by encoding it in the call, as without a store. */
int32_t krag_late_store_append(krag_late_store* s, int32_t n, const int32_t* passage_tok, const int32_t* passage_offsets,
                               const uint8_t* passage_keep, uint8_t* stored_out);
/* Drops ordinals n_ordinals and up (rolls an append back), freeing slabs left empty. */
int32_t krag_late_store_truncate(krag_late_store* s, int64_t n_ordinals);
/* Keeps the ordinals whose bit is set in alive_bitmap (bit o % 32 of word o / 32; n_ordinals must be the store's ordinal
 * count), renumbered 0 .. n_live - 1 in order; their rows move down on the device and slabs left empty are freed. */
int32_t krag_late_store_compact(krag_late_store* s, const uint32_t* alive_bitmap, int64_t n_ordinals);
/* ordinals, stored passages, stored rows and the slabs' device bytes (counted by krag_device_bytes); any pointer may be NULL */
int32_t krag_late_store_stats(const krag_late_store* s, int64_t* ordinals, int64_t* stored, int64_t* rows, int64_t* device_bytes);
/* krag_late_rerank with pair_source[j] >= 0 naming a stored ordinal (KRAG_E_INVALID when the store does not hold it) and
 * pair_source[j] < 0 naming passage ~pair_source[j] of the call (n_passages may be 0 when every pair names an ordinal). */
int32_t krag_late_rerank_stored(krag_embedder* e, const krag_late_store* s, int32_t n_queries, int32_t query_len, const int32_t* query_tok,
                                const int32_t* query_keys, int32_t n_passages, const int32_t* passage_tok, const int32_t* passage_offsets,
                                const uint8_t* passage_keep, const int32_t* pair_offsets, const int32_t* pair_source, int32_t top_k,
                                int32_t* out_pos, float* out_score);
/* The n_rows stored rows [n_rows, dim] of a stored ordinal (n_rows must be its row count).  Test hook. */
int32_t krag_debug_late_store_vectors(const krag_late_store* s, int64_t ordinal, float* out, int64_t n_rows);
int32_t krag_embedder_destroy(krag_embedder* e);

/* ------------------------------------------------- host-side text analysis (no GPU involved; ASCII input) */
/* The analysis chains the reference runs in native third-party code, for hosts that are not Python (a cgo host links the
 * same functions the Python host uses for ASCII text; kaito_b200/text.py is the Unicode-complete restatement and the spec).
 * krag_text_analyze: bm25s.tokenize(text, stopwords="english", stemmer=Snowball english) as used by
 *   BM25Retriever.from_defaults (hybrid_retriever.py:122-125): lower-case, \w\w+ tokens, 33 stop words dropped, Porter2 stems.
 *   Writes the stems separated by '\n' into out (if *out_len <= cap) and always reports the needed length and the token count.
 * krag_wordpiece_*: BertTokenizer (uncased) of the bge models (huggingface_local_embedding.py:34-53): BasicTokenizer +
 *   greedy longest-match WordPiece; vocab = the lines of vocab.txt joined by '\n'; encode_batch writes, per text,
 *   [CLS] ids[: max_len - 2] [SEP] (or the create_specials tokens) into out_ids[i * max_len ...] and its length into out_n[i] (texts are threaded). */
typedef struct krag_wordpiece krag_wordpiece;
int32_t krag_text_analyze(const char* text, int64_t len, char* out, int64_t cap, int64_t* out_len, int32_t* n_terms);
int32_t krag_wordpiece_create(const char* vocab, int64_t len, int32_t lower_case, krag_wordpiece** out);
/* the same with the unknown / first / last special tokens named (krag_wordpiece_create: "[UNK]", "[CLS]", "[SEP]"; MPNet:
 * "[UNK]", "<s>", "</s>"); each must be a line of vocab, else KRAG_E_INVALID.  Specials typed in a text are text. */
int32_t krag_wordpiece_create_specials(const char* vocab, int64_t len, int32_t lower_case, const char* unk_token,
                                       const char* cls_token, const char* sep_token, krag_wordpiece** out);
int32_t krag_wordpiece_encode_batch(const krag_wordpiece* w, int64_t n, const char* texts, const int64_t* offsets /*[n+1]*/,
                                    int32_t max_len, int32_t* out_ids /*[n * max_len]*/, int32_t* out_n /*[n]*/);
int32_t krag_wordpiece_destroy(krag_wordpiece* w);
/* krag_text_unigram_*: the SentencePiece Unigram tokeniser of XLM-RoBERTa models (bge-reranker-*) as the Rust `tokenizers`
 *   library runs a tokenizer.json, over tables the host parsed from it (kaito_b200/text.py, read_unigram_json):
 *   pieces = the model's pieces concatenated, piece i = pieces[piece_off[i] .. piece_off[i+1]) with log-probability
 *   scores[i]; unk_id; charsmap = the decoded normalizer precompiled_charsmap (charsmap_len 0: no normaliser); flags =
 *   1 (Replace " {2,}" -> " " after it) | 2 (WhitespaceSplit before Metaspace) | 4 (Metaspace prepend_scheme "first",
 *   else "always"); the added tokens likewise packed, with their ids and added_strip = 1 (lstrip) | 2 (rstrip).
 *   encode_batch writes the ids of text i without <s> / </s>, untruncated, into out_ids[i * cap ...] (at most cap of them)
 *   and their count into out_n[i] (which may exceed cap: call again with a larger cap). */
typedef struct krag_unigram krag_unigram;
int32_t krag_text_unigram_create(const char* pieces, const int64_t* piece_off /*[n_pieces+1]*/, const double* scores,
                                 int64_t n_pieces, int32_t unk_id, const char* charsmap, int64_t charsmap_len, int32_t flags,
                                 const char* added, const int64_t* added_off /*[n_added+1]*/, const int32_t* added_ids,
                                 const int32_t* added_strip, int32_t n_added, krag_unigram** out);
int32_t krag_text_unigram_encode_batch(const krag_unigram* u, int64_t n, const char* texts, const int64_t* offsets /*[n+1]*/,
                                       int32_t cap, int32_t* out_ids /*[n * cap]*/, int32_t* out_n /*[n]*/);
int32_t krag_text_unigram_destroy(krag_unigram* u);

/* ------------------------------------------------------------------- diagnostics */
/* C[M,N] = A[M,K] . B[N,K]^T + bias (+erf-GELU) (+residual) through K5's split-fp16 wgmma GEMM; host buffers.
 * N % 128 == 0, K % 64 == 0.  tile_n = 0: the tiles the forward would pick; 32, 64 or 128: 128 x tile_n tiles over the
 * whole K range.  reps > 0: the GEMM runs reps more times on the device operands and *ms_out gets the mean
 * time of one launch (CUDA events).  Test and probe hook. */
int32_t krag_debug_gemm_tf32(krag_ctx* ctx, int32_t M, int32_t N, int32_t K, const float* A, const float* B,
                             const float* bias, const float* residual, int32_t gelu, float* C_out, int32_t tile_n,
                             int32_t reps, float* ms_out);
/* The same through the single-plane fp16 GEMM of KRAG_PRECISION_FP16: A and B are rounded to fp16, one wgmma per step, fp32
 * accumulation and epilogue.  tile_n may also be 256 (N % 256 == 0).  Test and probe hook. */
int32_t krag_debug_gemm_f16(krag_ctx* ctx, int32_t M, int32_t N, int32_t K, const float* A, const float* B,
                            const float* bias, const float* residual, int32_t gelu, float* C_out, int32_t tile_n,
                            int32_t reps, float* ms_out);
/* Y = LayerNorm(A . B^T + bias (+residual)) * gamma + beta through K5's linear-layer dispatcher (for a handful of rows:
 * 128 x 32 split-K tiles + the reduce/LayerNorm kernel).  Test hook. */
int32_t krag_debug_linear_ln(krag_ctx* ctx, int32_t M, int32_t N, int32_t K, const float* A, const float* B,
                             const float* bias, const float* residual, const float* ln_gamma, const float* ln_beta,
                             float eps, float* Y_out);
/* Switch the dense kernel policy (KRAG_DENSE_*) of the context this index lives in.  Switching to KRAG_DENSE_TC_BF16
 * builds the index's bf16 shadow if it does not exist yet (one conversion pass over the fp32 rows); switching away
 * keeps the shadow unless release_shadow != 0.  Results never change: every mode returns exact fp32 distances.
 * A KRAG_ROWS_HOST index always keeps its bf16 rows (they are its device copy): release_shadow is ignored there. */
int32_t krag_index_set_dense_mode(krag_index* idx, int32_t dense_mode, int32_t release_shadow);
/* queries whose tensor-core result failed the exactness certificate and were re-run on the
 * exact scan kernel (process-wide counter) */
int64_t krag_tc_fallback_queries(void);
/* rows rescored from host memory by KRAG_ROWS_HOST searches (process-wide counter) */
int64_t krag_host_rows_fetched(void);
/* CUDA-event duration of the dominant dense kernel of the last search on this process
 * (kernel_id 1 = K1 exact scan; K2 main pass: 3 = TF32, 4 = bf16 shadow, 5 = bf16 high halves of the device rows,
 * 6 = device bf16 rows of a KRAG_ROWS_HOST index), with the algorithmic bytes and
 * flops of that launch -- bench.py's roofline line is computed from it. */
int32_t krag_last_dense_kernel(float* ms, int32_t* kernel_id, int64_t* algorithmic_bytes, int64_t* flops);
/* Figures of the last krag_index_compact (or redeal, see krag_redeal_begin) on this process: CUDA-event duration of the row-move phase (device moves and
 * the host-row memmoves they overlap), host-clock duration of the postings remap (0 if the index never committed),
 * live rows that changed position, and the bytes of the moved rows and term lists (each counted once). */
int32_t krag_last_compact(float* move_ms, float* postings_ms, int64_t* rows_moved, int64_t* bytes_moved);
/* Figures of the last commit on this process (krag_index_commit, or a commit_local / commit_global pair, reported by the
 * commit_global): host-clock duration of the whole commit, the part of it spent on the host computing idf, merged = 1
 * when the committed postings were merged with the changes (0: a full build, the first commit of an index and the one after
 * krag_index_load or krag_synth_fill), the postings written, and the term-list entries read to build them (those of the
 * rows added since the last commit when merged, every entry otherwise). */
int32_t krag_last_commit(float* total_ms, float* host_ms, int32_t* merged, int64_t* postings_written, int64_t* delta_entries);
/* test hook: rows [row0, row0 + n) of a device-resident index as stored, dim_padded 32-bit words per row (split rows where
 * dim_padded % 64 == 0, DESIGN.md section 4 K2) */
int32_t krag_debug_read_stored_rows(krag_index* idx, int64_t row0, int64_t n, float* out);
/* raw K2 output a[j][r] = |x_r|^2 - 2 x_r.q_j (TF32) for every row, [nq_pad][S] row-major;
 * call with out == NULL to query S and nq_pad.  Test hook for the tensor-core kernel; KRAG_E_UNSUPPORTED for
 * KRAG_ROWS_HOST indexes.  The same as krag_debug_tc_dump_pass(idx, KRAG_TC_PASS_TF32, ...). */
int32_t krag_debug_tc_dump(krag_index* idx, int32_t nq, const float* q, float* out, int64_t out_elems,
                           int64_t* S_out, int32_t* nq_pad_out);
/* the prune passes of K2 the test hooks below run (each the kernel instantiation the search itself uses) */
#define KRAG_TC_PASS_TF32 0        /* tf32 wgmma: on split rows their rebuilt fp32 values, else the plain fp32 rows */
#define KRAG_TC_PASS_BF16_SPLIT 1  /* bf16 wgmma on the high halves of split rows (kernel id 5) */
#define KRAG_TC_PASS_BF16_SHADOW 2 /* bf16 wgmma on the bf16 shadow (kernel id 4); KRAG_E_STATE when there is none */
#define KRAG_TC_PASS_BF16_HOST 3   /* bf16 wgmma on the device copy of a KRAG_ROWS_HOST index (kernel id 6) */
/* krag_debug_tc_dump for any prune pass: a[j][r] = |x_r|^2 - 2 x_r.q_j as that pass computes it, for every row (rows past
 * the end and tombstones included; the padding rows up to S are +inf) and every query column up to nq_pad (the NQ bucket
 * of nq: 64, 128 or 256; padded columns hold zero queries, so they return |x_r|^2).  Test hook. */
int32_t krag_debug_tc_dump_pass(krag_index* idx, int32_t pass, int32_t nq, const float* q, float* out, int64_t out_elems,
                                int64_t* S_out, int32_t* nq_pad_out);
/* one main prune pass of K2 over every row with caller-chosen thresholds: thr [nq_pad] (nq_pad = 64, 128 or 256, the NQ
 * bucket of nq; padded columns run zero queries with the thresholds given for them), the index's tombstones honoured.
 * counts_out [nq_pad] = rows with a < thr[j] (as the epilogue decides it), rows_out [nq_pad][cap] = the first
 * min(count, cap) of them in no particular order (entries past that undefined).  Test hook. */
int32_t krag_debug_tc_prune(krag_index* idx, int32_t pass, int32_t nq, const float* q, const float* thr, int32_t cap,
                            uint32_t* counts_out, uint32_t* rows_out);

#ifdef __cplusplus
}
#endif
#endif /* KAITO_RAG_H_ */
