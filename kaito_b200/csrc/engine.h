// engine.h -- internal launcher interface between the kernel translation units and api.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <functional>
#include <stdexcept>
#include <utility>
#include <vector>

#include "common.cuh"
namespace krag {

// device allocation failure with a message that says what was asked for and what was free (KRAG_E_OOM at the C ABI)
struct DevOom : std::runtime_error { using std::runtime_error::runtime_error; };

// bytes of device memory currently held through DevArray, process-wide (krag_device_bytes)
void count_device_bytes(int64_t delta);
int64_t device_bytes();

// Owning device buffer: the only code of the library that allocates or frees device memory.  Move-only; the destructor frees.
// An allocation that does not fit throws DevOom, saying how much was asked for and what was left.
template <class T>
struct DevArray {
    T* p = nullptr;
    int64_t cap = 0;

    DevArray() = default;
    DevArray(const DevArray&) = delete;
    DevArray& operator=(const DevArray&) = delete;
    DevArray(DevArray&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevArray& operator=(DevArray&& o) noexcept
    {
        if (this != &o) { release(); std::swap(p, o.p); std::swap(cap, o.cap); }
        return *this;
    }
    ~DevArray() { release(); }

    // a fresh buffer of exactly n elements; the old one is freed first
    void alloc(int64_t n)
    {
        release();
        p = allocate(n);
        cap = n;
    }
    // grow to at least n elements keeping the first `used` (copy-on-grow; krag_index_reserve avoids the copies for big corpora)
    void reserve(int64_t n, int64_t used, cudaStream_t st)
    {
        if (n <= cap) return;
        DevArray grown;
        grown.alloc(cap + cap / 2 > n ? cap + cap / 2 : n);
        if (p && used > 0) KRAG_CUDA(cudaMemcpyAsync(grown.p, p, sizeof(T) * (size_t)used, cudaMemcpyDeviceToDevice, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
        *this = std::move(grown);
    }
    // an exact-size buffer holding the first n elements, when one fits beside the current buffer; otherwise the capacity stays
    // (later growth reuses it).  Returns whether the buffer shrank.
    bool shrink(int64_t n, cudaStream_t st)
    {
        if (!p || n >= cap) return false;
        DevArray s;
        try {
            s.alloc(n);
        } catch (const DevOom&) {
            return false;
        }
        KRAG_CUDA(cudaMemcpyAsync(s.p, p, sizeof(T) * (size_t)n, cudaMemcpyDeviceToDevice, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
        *this = std::move(s);
        return true;
    }
    void release()
    {
        if (p) {
            cudaFree(p);
            count_device_bytes(-bytes());
        }
        p = nullptr;
        cap = 0;
    }
    int64_t bytes() const { return (int64_t)sizeof(T) * cap; }

private:
    static T* allocate(int64_t n)
    {
        void* q = nullptr;
        const size_t bytes = sizeof(T) * (size_t)n;
        const cudaError_t e = cudaMalloc(&q, bytes);
        if (e == cudaErrorMemoryAllocation) {
            cudaGetLastError();
            size_t free_b = 0, total_b = 0;
            cudaMemGetInfo(&free_b, &total_b);
            char msg[160];
            snprintf(msg, sizeof msg, "out of device memory (wanted %.2f GB, %.2f of %.2f GB free)", bytes / 1e9, free_b / 1e9,
                     total_b / 1e9);
            throw DevOom{msg};
        }
        KRAG_CUDA(e);
        count_device_bytes((int64_t)bytes);
        return static_cast<T*>(q);
    }
};

// bytes of pinned host memory currently held through HostArray, process-wide (krag_host_pinned_bytes)
void count_host_pinned_bytes(int64_t delta);
int64_t host_pinned_bytes();

// Owning pinned, device-mapped host buffer: the host counterpart of DevArray and the only code of the library that
// allocates, registers or frees pinned host memory.  `h` is the host address; `d` the address kernels read it through
// (zero-copy over the host link), taken from cudaHostGetDevicePointer, not assumed equal to `h`.  Move-only; the
// destructor frees.  An allocation that does not fit throws DevOom.
template <class T>
struct HostArray {
    T* h = nullptr;
    T* d = nullptr;
    int64_t cap = 0;

    HostArray() = default;
    HostArray(const HostArray&) = delete;
    HostArray& operator=(const HostArray&) = delete;
    HostArray(HostArray&& o) noexcept : h(o.h), d(o.d), cap(o.cap) { o.h = o.d = nullptr; o.cap = 0; }
    HostArray& operator=(HostArray&& o) noexcept
    {
        if (this != &o) { release(); std::swap(h, o.h); std::swap(d, o.d); std::swap(cap, o.cap); }
        return *this;
    }
    ~HostArray() { release(); }

    void alloc(int64_t n)
    {
        release();
        void* q = nullptr;
        const size_t bytes = sizeof(T) * (size_t)n;
        const cudaError_t e = cudaHostAlloc(&q, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
        if (e == cudaErrorMemoryAllocation) {
            cudaGetLastError();
            char msg[160];
            snprintf(msg, sizeof msg, "out of pinned host memory (wanted %.2f GB, %.2f GB already pinned by this process)", bytes / 1e9,
                     host_pinned_bytes() / 1e9);
            throw DevOom{msg};
        }
        KRAG_CUDA(e);
        h = static_cast<T*>(q);
        cap = n;
        count_host_pinned_bytes((int64_t)bytes);
        void* dp = nullptr;
        KRAG_CUDA(cudaHostGetDevicePointer(&dp, q, 0));
        d = static_cast<T*>(dp);
    }
    // grow to at least n elements keeping the first `used` (copy-on-grow on the host)
    void reserve(int64_t n, int64_t used)
    {
        if (n <= cap) return;
        HostArray grown;
        grown.alloc(cap + cap / 2 > n ? cap + cap / 2 : n);
        if (h && used > 0) memcpy(grown.h, h, sizeof(T) * (size_t)used);
        *this = std::move(grown);
    }
    // the host counterpart of DevArray::shrink
    bool shrink(int64_t n)
    {
        if (!h || n >= cap) return false;
        HostArray s;
        try {
            s.alloc(n);
        } catch (const DevOom&) {
            return false;
        }
        memcpy(s.h, h, sizeof(T) * (size_t)n);
        *this = std::move(s);
        return true;
    }
    void release()
    {
        if (h) {
            cudaFreeHost(h);
            count_host_pinned_bytes(-bytes());
        }
        h = d = nullptr;
        cap = 0;
    }
    int64_t bytes() const { return (int64_t)sizeof(T) * cap; }
};

// global ordinal of a local row: base + row * stride.  Contiguous shards (bench, one GPU) use stride 1; the multi-GPU
// service deals nodes round-robin (node o -> shard o % G, row o / G), so base = shard, stride = G and ordinals -- hence
// every tie-break -- are exactly the single-GPU insertion order.
struct OrdMap {
    uint32_t base, stride;
    __host__ __device__ __forceinline__ uint32_t operator+(uint32_t row) const { return base + row * stride; }
};

struct DeviceInfo {
    int device = 0;
    int sm_count = 132;
    int cc_major = 0, cc_minor = 0;
    size_t smem_optin = 0;
};

// CUDA-event bracket around the dominant dense kernel of the last search (roofline evidence):
// recorded on the launching stream; read back after the stream is synchronised.
void dense_timer_begin(cudaStream_t st, int kernel_id, int64_t algorithmic_bytes, int64_t flops);
void dense_timer_end(cudaStream_t st);
bool dense_timer_read(float* ms, int* kernel_id, int64_t* bytes, int64_t* flops);

// launch counter (bench.py reports gpu_launches from it)
void count_launch(int n = 1);
int64_t launch_count();

// ---- the dense rows of an index (dense_rows.cu): the rows in one of three layouts, and what is kept per row beside them
struct CompactPlan;
struct RedealRows;
// PLAIN: fp32 rows on the device (dpad % 64 == 32).  SPLIT: split rows on the device (split_rows.cuh, dpad % 64 == 0).
// HOST: fp32 rows in pinned host memory (KRAG_ROWS_HOST), with a bf16 copy and its residuals on the device.
enum class RowsLayout { PLAIN, SPLIT, HOST };
class DenseRows {
public:
    int dim = 0, dpad = 0;
    int64_t n = 0;                           // rows held
    RowsLayout layout = RowsLayout::PLAIN;   // decided once, by init

    void init(int dim, bool host_rows);
    bool host() const { return layout == RowsLayout::HOST; }
    bool split() const { return layout == RowsLayout::SPLIT; }
    // whether the rows keep a bf16 copy under this dense mode: host rows always; device rows as the KRAG_DENSE_TC_BF16
    // shadow, which stays once built unless release asks to drop it.  Whenever the copy exists it covers every row.
    bool keeps_bf16(int dense_mode, bool release = false) const;
    // room for `rows` rows; a bf16 copy that keeps_bf16 asks for and that does not exist yet is built from the rows held
    void reserve(int64_t rows, int dense_mode, cudaStream_t st);
    // rows [n, n + m): host fp32 rows [m, dim] (append) or the synthetic rows of global rows row_base + r (synth), with their
    // |x|^2, the running max, the bf16 copy and the stored layout.  The caller raises n once the rest of its update holds.
    void append(const float* vecs, int64_t m, int dense_mode, cudaStream_t st);
    void synth(int64_t m, int64_t row_base, uint64_t seed, int dense_mode, cudaStream_t st);
    // rows [row0, row0 + m) as fp32 [m, dim] on the host; read_stored: device rows as stored, [m, dpad]
    void read(int64_t row0, int64_t m, float* out) const;
    void read_stored(int64_t row0, int64_t m, float* out) const;
    // the bf16 shadow of device rows: built from the rows held when missing (on), or released (off); host rows keep their copy
    void set_shadow(bool on, cudaStream_t st);
    // row d <- row plan.src[d] in every array, in place; returns the bytes moved.  shrink: n = rows, the running max of
    // |x|^2 over them, and exact-size buffers where they fit; synchronises st.
    int64_t compact(const CompactPlan& plan, cudaStream_t st);
    void shrink(int64_t rows, cudaStream_t st);
    // a redeal's row view: these rows and the given term lists (null without)
    RedealRows redeal_rows(uint32_t* dlen, const int64_t* toff, const uint32_t* tid, const uint16_t* ttf) const;
    int64_t device_bytes() const;

    // what the kernels read
    const float* dev() const { return X.p; }        // device rows (PLAIN, SPLIT)
    const float* host_h() const { return Xp.h; }    // host rows: their host address (DMA source)
    const float* host_d() const { return Xp.d; }    // host rows: their mapped device address (zero-copy reads)
    const uint16_t* bf16() const { return Xh.p; }   // the bf16 copy [n, dpad], or null
    const float* res() const { return xres.p; }     // host rows: |x - bf16(x)| per row, rounded up
    const float* norms() const { return xnorm.p; }  // |x|^2 per row (K2 epilogue), from the fp32 rows
    const uint32_t* norm_max() const { return xn_max.p; }   // bits of max |x|^2 (K2 certificate)

private:
    DevArray<float> X;          // device rows [n, dpad], zero padded; split rows when SPLIT
    HostArray<float> Xp;        // host rows [n, dpad], zero padded
    DevArray<uint16_t> Xh;      // bf16 copy of the rows: optional shadow of device rows, always present for host rows
    DevArray<float> xres;       // host rows only
    DevArray<float> xnorm;
    DevArray<uint32_t> xn_max;  // [1]
    void derive(int64_t m, const uint64_t* gen_seed, int64_t row_base, cudaStream_t st);
    void reserve_bf16(int64_t elems, cudaStream_t st);
};

// device staging of the streamed exact scan, owned by the search slot
struct ScanStaging {
    float* buf[2];           // two chunks of chunk_rows rows (double buffering)
    int64_t chunk_rows;      // multiple of 32
    cudaStream_t copy;       // DMA stream
    cudaEvent_t copied[2], freed[2];
    uint64_t* fold;          // [2, batch, P]: running top P and the current chunk's
    float* q_sel;            // [256, dpad] uncertified queries of a K2 chunk
    uint64_t* k_sel;         // [256, P]
};
int64_t stream_scan_chunk_rows(int dpad);

// ---- K1: exact fp32 L2^2 scan + fused top-P (dense_scan.cu)
// q: device [batch, dpad] zero-padded.  part: workspace >= dense_scan_part_elems() u64.
// keys_out: device [batch, P], ascending, KEY_PAD padded, ordinals already global.  Device rows are scanned in place; host
// rows are copied in by DMA in chunks through sg (required then), each chunk's top P folded into the running list.  Exact.
size_t dense_scan_part_elems(const DeviceInfo& di, int P);
void launch_dense_scan(const DeviceInfo& di, const DenseRows& rows, const uint32_t* alive, const float* q, int batch, int P,
                       OrdMap ord_base, uint64_t* part, uint64_t* keys_out, cudaStream_t st, const ScanStaging* sg = nullptr);
void launch_bf16_residual(const float* X, int64_t n, int dpad, uint16_t* Xh, float* xres, cudaStream_t st);
int64_t host_rows_fetched();   // rows rescored from host memory, process-wide

// ---- K2: wgmma candidate generation + exact fp32 rescoring (dense_tc.cu)
// The prune operand of a K2 pass: every choice that follows from it is a row of TC_OPS or a branch of tc_pass (dense_tc.cu).
// The bf16 operands are KRAG_TC_PASS_* + 1.
enum TcOp { TC_OP_TF32, TC_OP_TF32S, TC_OP_BF16_SPLIT, TC_OP_BF16_SHADOW, TC_OP_BF16_HOST };
// the operand for these rows: shadow = prune on the bf16 shadow when there is one; tf32 = keep split rows on the TF32 pass
TcOp tc_operand(const DenseRows& rows, bool shadow, bool tf32);
bool dense_tc_supported(const DeviceInfo& di, int dpad);
bool dense_tc_wants(int64_t n_rows, int batch);   // size heuristics: is K2 the better kernel for this call?
bool dense_tc_serves(const DeviceInfo& di, const DenseRows& rows, TcOp op);   // can launch_dense_tc run op on these rows?
size_t dense_tc_workspace_bytes(const DeviceInfo& di, int64_t n_rows, int P, bool host_rows = false);
// |x|^2 per row (+ running max) maintained at index time for K2's epilogue and certificate
void launch_row_norms(const float* X, int64_t row0, int64_t n, int dpad, float* xnorm, uint32_t* xn_max_bits,
                      cudaStream_t st);
// For rows dense_tc_serves.  Returns false when the workspace or a tensor map does not fit (the caller runs K1 -- still GPU).
// Queries the certificate rejects are re-run on K1 inside: one by one on device rows, together through sg on host rows.
bool launch_dense_tc(const DeviceInfo& di, const DenseRows& rows, TcOp op, const uint32_t* alive, const float* q, int batch,
                     int P, OrdMap ord_base, void* workspace, size_t workspace_bytes, uint64_t* part, const ScanStaging* sg,
                     uint64_t* keys_out, cudaStream_t st);
void launch_f32_to_bf16(const float* in, uint16_t* out, int64_t n_elems, cudaStream_t st);
int64_t dense_tc_fallback_queries();   // queries re-run on K1 because the exactness certificate failed
// diagnostics (tests only): one prune pass of K2 on operand op over every tile of the rows, in the production instantiation.
// cap == 0: the DUMP instantiation writes a[j][r] = |x_r|^2 - 2 x_r.q_j for ALL rows and NQ_pad query columns to w.dump
// [NQ_pad][S] (rows past n_rows: +inf); cap > 0: the main pass appends the alive rows with a < w.thr[j] to w.cand_rows
// [NQ_pad][cap] and counts them in w.cand_count [NQ_pad].  w is carved by dense_tc_debug_carve (base == nullptr: size only).
struct TcDebugWs { uint16_t* q_bf16; float* dump; float* thr; uint32_t* cand_count; uint32_t* cand_rows; };
size_t dense_tc_debug_carve(TcDebugWs* w, unsigned char* base, int64_t n_rows, int dpad, int nq, int cap, int64_t* S_out,
                            int* nq_pad_out);
bool dense_tc_debug_pass(const DeviceInfo& di, const DenseRows& rows, TcOp op, const uint32_t* alive, const float* q, int nq,
                         const TcDebugWs& w, int cap, cudaStream_t st);

// ---- merge / fuse (merge_fuse.cu)
// per query: n_lists lists of list_len keys (element (l,i) at in[b*batch_stride + l*list_stride + i]) -> the P smallest
// only_flag != null: queries whose flag is 0 are left untouched
void launch_merge(const uint64_t* keys_in, int n_lists, int list_len, int batch, int P, int64_t list_stride,
                  int64_t batch_stride, uint64_t* keys_out, cudaStream_t st, const uint64_t* thr_hint = nullptr,
                  const uint32_t* only_flag = nullptr);
// peer-memory exchange: push local lists [nl, batch, P] into every rank's mailbox, then merge G*P -> P locally
size_t p2p_mailbox_words(int world, int nl, int max_batch, int max_P);
void launch_p2p_exchange_merge(uint64_t* const* d_mailboxes, uint64_t* own_mailbox, int rank, int world, int64_t slot_words,
                               unsigned long long seq, int nl, int batch, int P, const uint64_t* local, uint64_t* merged,
                               cudaStream_t st);
void launch_bitmap_and(uint32_t* dst, const uint32_t* other, int64_t words, cudaStream_t st);
// append zero-score fillers to short BM25 lists (bm25s argpartition semantics)
void launch_bm25_fill(uint64_t* keys /*[batch,P]*/, int batch, int P, const uint32_t* alive, int64_t n_rows,
                      OrdMap ord_base, cudaStream_t st);
void launch_fuse(int batch, int P, int k, const uint64_t* dense_keys, const uint64_t* bm25_keys, double w_v, double w_t,
                 int mode, const uint32_t* allow, double* out_final, float* out_dense, float* out_sparse,
                 int32_t* out_rank, int64_t* out_ord, int32_t* out_count, cudaStream_t st);

// ---- K3: BM25 (bm25.cu)
constexpr int BM25_SUB_DOCS = 2048;      // doc range of one tile-index column = one warp's shared-memory accumulator (K3)
constexpr int BM25_SUBS_PER_TILE = 8;
constexpr int BM25_TILE_DOCS = BM25_SUB_DOCS * BM25_SUBS_PER_TILE;   // doc range of one CTA in the legacy kernel (safety net)
struct Postings {
    DevArray<int64_t> off;     // [vocab+1]
    DevArray<uint32_t> doc;    // [nnz] local rows ascending inside a term
    DevArray<uint16_t> tf;     // [nnz] term frequency of the posting: an incremental commit rescores from it (K3 never reads it)
    DevArray<float> score;     // [nnz]
    int64_t vocab = 0, nnz = 0;
    // tile index: for terms with more than BM25_RARE_MAX postings, the offset (relative to off[t]) of the
    // first posting whose doc lies in each BM25_SUB_DOCS-sized doc range; removes per-query searches.  Terms below the
    // threshold get the same kind of row built per batch by bm25_resolve_kernel (a row costs 4 B per sub-tile, more than
    // the postings of a short list)
    DevArray<int32_t> tile_slot;    // [vocab]  slot of a frequent term, -1 for the others
    DevArray<uint32_t> tile_off;    // [n_slots][n_tiles + 1]
    int64_t n_slots = 0, n_tiles = 0;   // n_tiles = number of BM25_SUB_DOCS ranges
};
constexpr int BM25_RARE_MAX = 2048;
void launch_df_histogram(const uint32_t* term_ids, const uint32_t* entry_doc, const uint32_t* alive, int64_t nnz,
                         uint32_t* df, cudaStream_t st);
// entry_doc[i - term_offsets[row0]] = d for the entries i of rows d in [row0, row0 + n_docs)
void launch_expand_entry_doc(const int64_t* term_offsets, int64_t n_docs, uint32_t* entry_doc, cudaStream_t st, int64_t row0 = 0);
// score(t, d) = f32(f64(idf[t]) * tf / (k1 * ((1 - b) + b * dl / avgdl) + tf)), k1 = 1.5, b = 0.75, left to right as Python
// evaluates it, every operation correctly rounded and none contracted: the full build and the incremental merge both use it
__device__ __forceinline__ float bm25_posting_score(float idf, uint32_t tf, uint32_t dl, double avgdl)
{
    const double k1 = 1.5, b = 0.75;
    const double tfd = (double)tf;
    double t1 = __dmul_rn(b, (double)dl);
    double t2 = __ddiv_rn(t1, avgdl);
    double t3 = __dadd_rn(__dsub_rn(1.0, b), t2);
    double t4 = __dmul_rn(k1, t3);
    double t5 = __dadd_rn(t4, tfd);
    double tfc = __ddiv_rn(tfd, t5);
    return __double2float_rn(__dmul_rn((double)idf, tfc));
}
// df [vocab] (device) -> off [vocab + 1] = exclusive scan (int64), with a host copy when h_off != null; synchronises st
void df_offsets(const uint32_t* df, int64_t vocab, DevArray<int64_t>& off, std::vector<int64_t>* h_off, cudaStream_t st);
// tile index of postings with offsets off: slots of the frequent terms and the boundary table, to be filled; or, for
// postings without entries, no slot at all
void prepare_tile_index(const int64_t* off, int64_t vocab, int64_t n_rows, Postings& out, cudaStream_t st);
void empty_tile_index(int64_t vocab, int64_t n_rows, Postings& out);
// The live entries of CSR-by-doc arrays sorted by term, documents ascending inside a term, one term range at a time:
// per_range(p_base, m, keys, vals) gets postings [p_base, p_base + m) of the offsets h_off (host copy of the live df's
// exclusive scan) as term ids and (doc << 16 | tf), valid until it returns.  Synchronises st at the end.
using TermRangeFn = std::function<void(int64_t p_base, int64_t m, const uint32_t* keys, const uint64_t* vals)>;
void sort_entries_by_term(const uint32_t* term_ids, const uint16_t* term_tf, const uint32_t* entry_doc, const uint32_t* alive,
                          int64_t nnz, int64_t vocab, const std::vector<int64_t>& h_off, const TermRangeFn& per_range,
                          cudaStream_t st);
// builds postings from CSR-by-doc arrays; idf is a device array [vocab] computed on the host (glibc log)
void build_postings(const uint32_t* term_ids, const uint16_t* term_tf, const uint32_t* entry_doc,
                    const uint32_t* doc_len, const uint32_t* alive, int64_t nnz, int64_t vocab, const float* idf,
                    double avgdl, int64_t n_docs_rows, Postings& out, cudaStream_t st);
size_t bm25_part_elems(int64_t n_rows, int batch, int P);
size_t bm25_resolve_bytes(int64_t n_rows, int n_terms_total);   // size of launch_bm25's resolve_ws
void launch_bm25(const DeviceInfo& di, const Postings& post, int64_t n_rows, const uint32_t* alive,
                 const uint32_t* q_terms, const int32_t* q_term_offsets, int n_terms_total, void* resolve_ws, int batch, int P,
                 OrdMap ord_base, uint64_t* part, uint64_t* keys_out, cudaStream_t st);

// ---- incremental postings (postings_merge.cu).  The postings of a commit stay the *base* of the next one: for each term,
// the rows below base_rows that were alive then, ascending.  Rows never come back to life and rows added since have higher
// numbers, so a term's new list is its base list without the rows dead now, followed by its live new rows.
struct SurvivorCounts {
    DevArray<uint32_t> per_term;    // [vocab] live postings of each term's base list
    DevArray<int64_t> before;       // [vocab + 1] exclusive scan of per_term
    DevArray<int64_t> block_off;    // [blocks of the base postings] live base postings before each block
};
// survivors of base postings `base` (alive == null: all live) counted per term, for the new vocab (>= every base term + 1)
void count_survivors(const Postings& base, const uint32_t* alive, int64_t vocab, SurvivorCounts& sc, cudaStream_t st);
// writes the survivors of `base` into out (allocated): survivor k of term t (base order) lands at out_off[t] + k.
// Rescored (doc_len, idf, avgdl) when rank == null; otherwise doc -> rank[doc] with tf and score copied.
void write_survivors(const Postings& base, const uint32_t* alive, const SurvivorCounts& sc, const int64_t* out_off,
                     const uint32_t* rank, const uint32_t* doc_len, const float* idf, double avgdl, Postings& out, cudaStream_t st);
// delta postings (term ids keys, (doc << 16 | tf) vals) [q_base, q_base + m) of the delta offsets delta_off: delta posting q of
// term t lands at out_off[t] + survivors(t) + (q - delta_off[t]), rescored
void write_delta(const uint32_t* keys, const uint64_t* vals, int64_t q_base, int64_t m, const int64_t* delta_off,
                 const SurvivorCounts& sc, const int64_t* out_off, const uint32_t* doc_len, const float* idf, double avgdl,
                 Postings& out, cudaStream_t st);
// fills the tile index prepared by prepare_tile_index from out.off / out.doc
void fill_tile_index(Postings& out, cudaStream_t st);
// (live rows, sum of their doc_len) over rows [0, n_rows)
void live_doc_stats(const uint32_t* doc_len, const uint32_t* alive, int64_t n_rows, int64_t* n_live, int64_t* total_len,
                    cudaStream_t st);
void launch_add_u32(const uint32_t* a, const uint32_t* b, int64_t n, uint32_t* out, cudaStream_t st);
void launch_rank_of_rows(const uint32_t* src, int64_t n_live, uint32_t* rank, cudaStream_t st);

// ---- compaction (compact.cu): tombstoned rows removed in place, live rows keep their order
constexpr int64_t COMPACT_STAGE_BYTES = (int64_t)32 << 20;   // staging of windows whose source and destination overlap
constexpr int64_t COMPACT_TERM_BYTES = sizeof(uint32_t) + sizeof(uint16_t);   // one CSR entry: term id + tf
struct CompactPlan {
    int64_t n_rows = 0, n_live = 0;
    int64_t first = 0;                  // first destination row that moves (= the first dead row); rows before it stay
    DevArray<uint32_t> src;             // [n_live] source row of destination row d (ascending)
    std::vector<uint32_t> h_src;
    DevArray<int64_t> toff_new;         // [n_live + 1] term-list offsets after compaction (hybrid indexes)
    std::vector<int64_t> h_toff_old, h_toff_new;
    DevArray<unsigned char> stage;      // COMPACT_STAGE_BYTES, or the longest moved term list if that is larger
};
// ranks of the live rows (popcount prefix over the alive words) and, with toff, the new term-list offsets.  Allocates every
// temporary of the compaction, so an allocation failure happens before any row has moved.
void compact_plan(const uint32_t* alive, int64_t n_rows, const int64_t* toff, CompactPlan& plan, cudaStream_t st);
// rows of row_bytes (a multiple of 4) at base: row d <- row src[d], in place; returns the bytes of the rows that moved
int64_t compact_rows(void* base, int64_t row_bytes, const CompactPlan& plan, cudaStream_t st);
// CSR term lists (tid / ttf) in place under toff_old -> plan.toff_new; returns the bytes of the entries that moved
int64_t compact_terms(uint32_t* tid, uint16_t* ttf, const int64_t* toff_old, const CompactPlan& plan, cudaStream_t st);
// *max_bits = bits of max x[i] over [0, n), x >= 0 (the K2 certificate's max |x|^2, as row_norms_kernel keeps it)
void launch_max_bits(const float* x, int64_t n, uint32_t* max_bits, cudaStream_t st);

// ---- redeal (compact.cu): G round-robin shards (shard s holds global ordinals s, s + G, ...) compacted together.  Live row
// with old ordinal o gets the new ordinal rank(o) (live ordinals below o) and moves to shard rank % G, row rank / G.  Moves
// run in windows [R0, R1) of new ordinals, ascending from the first dead ordinal; rank(o) <= o, so every row a shard reads
// in a window or later lies at or above R0 and every row it wrote before lies below: packing a window before unpacking it
// overwrites no row that is still to be read.  Term lists go to new arrays of their exact size.
// Row payload: 16 B header (u32 destination row, u32 term count, i64 entry offset inside the sender's chunk for this
// destination), 16 B scalars (u32 doc_len, f32 |x|^2, f32 xres, 0), the fp32 row [dpad], the bf16 row [dpad] if present.
// Entry payload: 8 B (u32 term id, u32 tf).
constexpr int64_t REDEAL_HEAD_BYTES = 32;
constexpr int64_t REDEAL_ENTRY_BYTES = 8;
struct RedealRows {
    float* x;            // fp32 rows (device, or the mapped address of pinned host rows)
    uint16_t* xh;        // bf16 rows or null
    float* xres;         // or null
    float* xnorm;
    uint32_t* dlen;      // or null (no term lists)
    const int64_t* toff; // or null
    const uint32_t* tid;
    const uint16_t* ttf;
    int dpad;
};
struct RedealPlan {
    int G = 1, s = 0;
    int64_t words = 0, n_rows = 0, window_rows = 1;
    int64_t n_live = 0;          // live rows over all shards
    int64_t first = 0;           // first dead ordinal (new ordinals below it do not move)
    int64_t n_windows = 0, row_bytes = 0;
    int64_t n_send = 0;          // this shard's rows that move
    int64_t n_new = 0, j_first = 0;   // rows of this shard afterwards; rows [0, j_first) stay where they are
    DevArray<uint32_t> rank;     // [n_rows] new ordinal of each live local row
    DevArray<uint32_t> send_key, send_row;   // [n_send] window * G + destination, local row: in send order
    DevArray<int64_t> send_ent;  // [n_send + 1] entry offsets in send order
    DevArray<int64_t> seg_ent;   // [n_windows * G + 1] send_ent at the start of each (window, destination) segment
    std::vector<int64_t> send_rows, send_ents, recv_rows;   // [n_windows][G]
    std::vector<int64_t> seg_row;                            // [n_windows * G + 1]
    // receiving side (redeal_prepare)
    std::vector<int64_t> recv_ents, ent_base;                // [n_windows][G], [n_windows + 1]
    DevArray<int64_t> recv_row_disp, recv_ent_disp;          // [n_windows][G + 1], [n_windows][G]
    DevArray<int64_t> lens, toff_new;                        // [max window rows], [n_new + 1]
    DevArray<uint32_t> tid_new;
    DevArray<uint16_t> ttf_new;
    DevArray<unsigned char> scan_tmp;
    size_t scan_bytes = 0;
    int64_t j0(int64_t k) const;      // first destination row of window k on this shard
};
// the plan from every shard's alive bitmap (host [G][words]; bits past a shard's rows are 0), this shard's term offsets (or
// null) and the window width; synchronises st
void redeal_plan(const uint32_t* h_alive, int G, int s, int64_t words, int64_t n_rows, const int64_t* toff, bool has_xh, int dpad,
                 int64_t window_rows, RedealPlan& p, cudaStream_t st);
// the receiving side: the senders' entry counts [n_windows][G], the new term arrays (rows that stay copied over); synchronises st
void redeal_prepare(const int64_t* recv_ents, const int64_t* toff, const uint32_t* tid, const uint16_t* ttf, RedealPlan& p,
                    cudaStream_t st);
// window k: this shard's rows into rows / ents (send order), and the received rows / ents into place
void redeal_pack(const RedealRows& v, const RedealPlan& p, int64_t k, void* rows, void* ents, cudaStream_t st);
void redeal_unpack(const RedealRows& v, RedealPlan& p, int64_t k, const void* rows, const void* ents, cudaStream_t st);

// ---- K5: BERT encoder forward (embed.cu)
struct BertConfig;
struct Embedder;
Embedder* embedder_create(const DeviceInfo& di, const BertConfig& cfg);
void embedder_load(Embedder* e, const char* name, const float* data, int64_t n);
void embedder_finalize(Embedder* e);
void embedder_destroy(Embedder* e);
int embedder_hidden(const Embedder* e);
enum { EMB_POOL_CLS = 0, EMB_POOL_MEAN = 1 };   // = KRAG_POOL_CLS / KRAG_POOL_MEAN
void embedder_set_pooling(Embedder* e, int mode);
// test hook: false runs the last layer over every token under CLS pooling too (same results)
void embedder_set_cls_rows_only(Embedder* e, bool on);
// arithmetic of every GEMM / attention product of the forward: split fp16 operands, three MMAs (fp32-accurate), or the hi
// planes alone, one MMA; accumulation, residual stream, LayerNorm, softmax and the head are fp32 in both
enum { EMB_PREC_FP32 = 0, EMB_PREC_FP16 = 1 };   // = KRAG_PRECISION_FP32 / KRAG_PRECISION_FP16
void embedder_set_precision(Embedder* e, int mode);
// first position row of every sequence (RoBERTa / XLM-R: pad_token_id + 1); token i of a sequence takes row off + i
void embedder_set_position_offset(Embedder* e, int off);
// MPNet: the bucket of MPNetEncoder.relative_position_bucket (32 buckets, max distance 128) the attention kernel applies at
// rel = key - query (the distance clamped to +-128 first); host-only
int relative_bucket(int rel);
// rotary encoders (nomic-bert): positions rotate Q and K instead of a position table; base = the rotary base (0: off).
// Called before finalize.
void embedder_set_rotary(Embedder* e, float base);
// the fp32 (cos, sin) of the rotary angle fp32(pos) * inv_freq[i], inv_freq[i] = 1 / base^(2i / dh) in fp32, for i < dh / 2
// (what the QKV epilogue applies; transformers' default RoPE); host-only
void rotary_cos_sin(float base, int dh, int pos, float* cos_out, float* sin_out);
void embedder_forward(Embedder* e, int batch, const int32_t* tok_ids, const int32_t* tok_offsets, float* out_host,
                      float* out_dev = nullptr, int ld_out = 0, cudaStream_t consumer = nullptr);
// cross-encoder reranking (classifier head loaded): scores of sentence pairs, top_k per query (see embed.cu)
enum { EMB_ACT_SIGMOID = 0, EMB_ACT_IDENTITY = 1 };   // = KRAG_RERANK_SIGMOID / KRAG_RERANK_IDENTITY
constexpr int RERANK_MAX_CANDIDATES = 300;           // pairs per query (= KRAG_MAX_TOP_K)
constexpr int RERANK_MAX_TOKENS = 65536;             // tokens per forward of a rerank call
void embedder_rerank(Embedder* e, int n_queries, const int32_t* pair_off, const int32_t* tok_ids, const int32_t* tok_off,
                     const int32_t* seg_b, int act, int top_k, int32_t* out_pos, float* out_score);
// late interaction (ColBERT): the hidden -> dim projection (linear.weight [dim][hidden], no bias; before finalize), the unit
// token vectors of packed sequences (kv_len: keys per sequence, or null), and MaxSim reranking (see embed.cu)
void embedder_set_late_interaction(Embedder* e, int dim, const float* weight, int64_t n);
void embedder_late_vectors(Embedder* e, int batch, const int32_t* tok_ids, const int32_t* tok_off, const int32_t* kv_len, float* out_host);
void embedder_late_rerank(Embedder* e, int n_queries, int q_rows, const int32_t* q_tok, const int32_t* q_kv, int n_pass, const int32_t* p_tok,
                          const int32_t* p_off, const uint8_t* p_keep, const int32_t* pair_off, const int32_t* pair_pass, int top_k,
                          int32_t* out_pos, float* out_score);
// Stores of passage token vectors (kept rows only, fp32, per ordinal in device slabs) filled from a late-interaction
// embedder; their slabs share the embedder's budget of device bytes.  late_store_rerank: pair_src >= 0 names a stored
// ordinal, < 0 passage ~pair_src of the call (see embed.cu)
struct LateStore;
void embedder_set_store_budget(Embedder* e, int64_t bytes);
LateStore* late_store_create(Embedder* e);
void late_store_destroy(LateStore* s);
void late_store_append(LateStore* s, int n, const int32_t* tok, const int32_t* off, const uint8_t* keep, uint8_t* stored_out);
void late_store_truncate(LateStore* s, int64_t n);
void late_store_compact(LateStore* s, const uint32_t* alive, int64_t n);
void late_store_stats(const LateStore* s, int64_t* ordinals, int64_t* stored, int64_t* rows, int64_t* bytes);
void late_store_vectors(const LateStore* s, int64_t ordinal, float* out_host, int64_t n_rows);
void late_store_rerank(Embedder* e, const LateStore* s, int n_queries, int q_rows, const int32_t* q_tok, const int32_t* q_kv, int n_pass,
                       const int32_t* p_tok, const int32_t* p_off, const uint8_t* p_keep, const int32_t* pair_off, const int32_t* pair_src,
                       int top_k, int32_t* out_pos, float* out_score);
// A fp32 matrix carried as two fp16 planes: v = hi + lo * 2^-11 (see embed.cu: split operands of the K5 GEMMs)
struct SplitMat { uint16_t* hi; uint16_t* lo; };
void launch_split_f16(const float* in, uint16_t* hi, uint16_t* lo, int64_t n /* % 8 == 0 */, cudaStream_t st);
// Linear layer on split operands: C = A . B^T + bias (+GELU) (+residual), fp32-accurate (three fp16 wgmma per step);
// outputs: fp32 C and / or the split planes of C; with ln_g the row LayerNorm of that goes to Y / Y planes (C is scratch).
// Tile width bn of the 128 x bn output tiles, K slices (splits > 1: fp32 partials in ws + a reduce kernel), and whether the
// small-M path (bn 32 / 64 / 128, split-K, workspace) or the large-M one (128 x 128, whole K) runs.
// planes = 1: the single-plane product (A.lo, B.lo and the lo outputs are not touched; one fp16 wgmma per step, fp32
// accumulation), whose large-M path also has 128 x 256 tiles.
struct GemmPlan { int bn; int splits; bool small_m; };
// Epilogue variants of a linear layer (compile-time kernel variants, see gemm_f16s_kernel): EP_PLAIN (BERT), EP_ROPE (rotary
// positions on the Q and K columns of a QKV projection whose weight rows were permuted per head), EP_SWIGLU (gated FFN1 on
// interleaved up / gate rows: N = 2 * inter columns in, inter out).
enum { EP_PLAIN = 0, EP_ROPE = 1, EP_SWIGLU = 2 };
struct EpiArgs {
    int mode;                 // EP_*
    const float* rope;        // EP_ROPE: [positions][half] (cos, sin) pairs, fp32
    const int32_t* pos;       // EP_ROPE: position of every row of A
    int rope_cols;            // EP_ROPE: columns [0, rope_cols) are rotated (2 * hidden: Q and K)
    int half;                 // EP_ROPE: head_dim / 2
};
// the plan launch_linear picks for M rows: 128 x 128 tiles, or 128 x BN split-K tiles for few activation tiles
GemmPlan linear_plan(const DeviceInfo& di, int M, int N, int K, bool ln, bool have_ws, size_t ws_floats, int planes = 2);
// plan = null: linear_plan(M, ...); ws = split-K workspace (may be null); ep = null: EP_PLAIN (EP_ROPE / EP_SWIGLU take no
// LayerNorm, residual or GELU; EP_SWIGLU's C / C planes are [M][N / 2])
void launch_linear(const DeviceInfo& di, const SplitMat& A, const SplitMat& B, int M, int N, int K, const float* bias, const float* residual,
                   bool gelu, float* C, uint16_t* C_hi, uint16_t* C_lo, const float* ln_g, const float* ln_b, float eps, float* Y,
                   uint16_t* Y_hi, uint16_t* Y_lo, float* ws, size_t ws_floats, cudaStream_t st, const GemmPlan* plan = nullptr,
                   int planes = 2, const EpiArgs* ep = nullptr);
// test hook: fp32 device operands, split on the fly, then the path above.  tile_n = 0: launch_linear's own plan; 32, 64 or
// 128 (256 with planes = 1): that tile width over the whole K range.  reps > 0: the GEMM is launched reps more times between two CUDA
// events and *ms gets the mean time of one launch.
void launch_linear_f32(const DeviceInfo& di, const float* A, const float* B, int M, int N, int K, const float* bias, const float* residual,
                       bool gelu, float* C, const float* ln_g, const float* ln_b, float eps, float* Y, float* ws, size_t ws_floats,
                       cudaStream_t st, int tile_n = 0, int reps = 0, float* ms = nullptr, int planes = 2);

// ---- synthetic data (synth.cu)
void launch_synth_dense(float* X, int64_t n, int d, int dpad, int64_t row_base, uint64_t seed, cudaStream_t st);
// two-pass: lengths -> offsets (host scan by caller via cub) -> fill
void synth_sparse(int64_t n, int64_t row_base, uint64_t seed, int64_t vocab, DevArray<int64_t>& term_offsets,
                  DevArray<uint32_t>& term_ids, DevArray<uint16_t>& term_tf, DevArray<uint32_t>& doc_len, int64_t* nnz_out,
                  cudaStream_t st);

}  // namespace krag
