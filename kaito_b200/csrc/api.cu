// api.cu -- the C ABI of libkaito_rag.so (include/kaito_rag.h): context, index shards,
// host-buffer search entry points and the device-pointer stage API.
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <sys/stat.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/kaito_rag.h"
#include "common.cuh"
#include "embed_config.h"
#include "engine.h"

namespace krag {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
static std::atomic<int64_t> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int64_t launch_count() { return g_launches.load(std::memory_order_relaxed); }
static std::atomic<int64_t> g_device_bytes{0};
void count_device_bytes(int64_t delta) { g_device_bytes.fetch_add(delta, std::memory_order_relaxed); }
int64_t device_bytes() { return g_device_bytes.load(std::memory_order_relaxed); }
static std::atomic<int64_t> g_host_pinned_bytes{0};
void count_host_pinned_bytes(int64_t delta) { g_host_pinned_bytes.fetch_add(delta, std::memory_order_relaxed); }
int64_t host_pinned_bytes() { return g_host_pinned_bytes.load(std::memory_order_relaxed); }

// "last dense kernel" diagnostics (krag_last_dense_kernel, read by bench.py).  Process-wide and last-writer-wins: with
// concurrent searches the numbers describe one of them; the mutex only keeps the record itself consistent.
static std::mutex g_t_mu;
static cudaEvent_t g_t0 = nullptr, g_t1 = nullptr;
static int g_t_kernel = 0;
static int64_t g_t_bytes = 0, g_t_flops = 0;
static bool g_t_valid = false;
void dense_timer_begin(cudaStream_t st, int kernel_id, int64_t bytes, int64_t flops)
{
    std::lock_guard<std::mutex> lk(g_t_mu);
    if (!g_t0) { cudaEventCreate(&g_t0); cudaEventCreate(&g_t1); }
    g_t_kernel = kernel_id; g_t_bytes = bytes; g_t_flops = flops; g_t_valid = false;
    cudaEventRecord(g_t0, st);
}
void dense_timer_end(cudaStream_t st)
{
    std::lock_guard<std::mutex> lk(g_t_mu);
    cudaEventRecord(g_t1, st);
    g_t_valid = true;
}
bool dense_timer_read(float* ms, int* kernel_id, int64_t* bytes, int64_t* flops)
{
    std::lock_guard<std::mutex> lk(g_t_mu);
    if (!g_t_valid || cudaEventSynchronize(g_t1) != cudaSuccess || cudaEventElapsedTime(ms, g_t0, g_t1) != cudaSuccess) return false;
    *kernel_id = g_t_kernel; *bytes = g_t_bytes; *flops = g_t_flops;
    return true;
}

struct ApiError { int32_t code; std::string msg; };
#define KRAG_REQUIRE(cond, code, msg)                      \
    do {                                                   \
        if (!(cond)) throw ::krag::ApiError{(code), (msg)}; \
    } while (0)

template <class F>
static int32_t guarded(F&& f)
{
    try {
        f();
        return KRAG_OK;
    } catch (const ApiError& e) {
        set_error(e.msg);
        return e.code;
    } catch (const CudaError& e) {
        char buf[512];
        snprintf(buf, sizeof buf, "CUDA error %d (%s) at %s:%d: %s", (int)e.e, cudaGetErrorString(e.e), e.file, e.line, e.what);
        set_error(buf);
        cudaGetLastError();
        return e.e == cudaErrorMemoryAllocation ? KRAG_E_OOM : KRAG_E_CUDA;
    } catch (const DevOom& e) {
        set_error(e.what());
        return KRAG_E_OOM;
    } catch (const std::bad_alloc&) {
        set_error("host allocation failed");
        return KRAG_E_OOM;
    } catch (const std::exception& e) {
        set_error(e.what());
        return KRAG_E_INVALID;
    }
}

// per-call search workspace
struct Slot {
    cudaStream_t st = nullptr;
    DevArray<float> q;
    DevArray<uint32_t> terms;
    DevArray<int32_t> toff;
    DevArray<uint64_t> dense_keys, bm25_keys, part;
    DevArray<unsigned char> tc_ws, bm25_res;
    DevArray<uint32_t> allow;
    DevArray<double> out_final;
    DevArray<float> out_dense, out_sparse;
    DevArray<int32_t> out_rank, out_count;
    DevArray<int64_t> out_ord;
    std::vector<float> hq;  // padded query staging
    // streamed exact scan over host-resident rows (created on first use)
    DevArray<float> stage;
    DevArray<uint64_t> fold, k_sel;
    DevArray<float> q_sel;
    cudaStream_t copy_st = nullptr;
    cudaEvent_t copied[2] = {nullptr, nullptr}, freed[2] = {nullptr, nullptr};
    // recorded after the work of each call that used the slot, on the stream that work went to (SlotLease)
    cudaEvent_t done = nullptr;
    ~Slot()
    {
        for (cudaEvent_t e : {copied[0], copied[1], freed[0], freed[1], done}) if (e) cudaEventDestroy(e);
        if (copy_st) cudaStreamDestroy(copy_st);
        if (st) cudaStreamDestroy(st);
    }
};

}  // namespace krag

using namespace krag;

struct krag_ctx {
    DeviceInfo di;
    krag_config cfg;
    std::mutex mu;
    std::condition_variable cv;
    std::vector<std::unique_ptr<Slot>> all_slots;
    std::vector<Slot*> free_slots;
    cudaStream_t admin = nullptr;  // mutation / build stream
    ~krag_ctx() { if (admin) cudaStreamDestroy(admin); }
};

// what krag_index_commit_local leaves for krag_index_commit_global: valid for one index state (epoch) and vocab
struct CommitPrep {
    bool valid = false, merge = false;
    int64_t vocab = 0, epoch = 0;
    DevArray<uint32_t> entry_doc;   // row of each entry read: every entry (full build) or those of rows >= committed_rows (merge)
    int64_t e0 = 0;                 // first entry read
    SurvivorCounts sc;              // merge: live base postings per term
    DevArray<uint32_t> delta_df;    // merge: live entries of rows >= committed_rows per term
    double ms = 0.0;                // host-clock time spent preparing
};

struct krag_index {
    krag_ctx* ctx = nullptr;
    std::string name;
    std::shared_mutex mu;
    DenseRows rows;                 // the dense shard; rows.n is the index's row count
    int64_t n_live = 0;
    std::vector<uint32_t> alive_h;
    DevArray<uint32_t> alive_d;
    bool has_dead = false;
    std::vector<uint64_t> node_ids;
    std::unordered_map<uint64_t, int64_t> id2row;
    // sparse raw (CSR by doc)
    bool has_sparse = false;
    DevArray<int64_t> toff;
    DevArray<uint32_t> tid;
    DevArray<uint16_t> ttf;
    DevArray<uint32_t> dlen;
    int64_t nnz = 0;
    uint32_t max_term_id = 0;       // largest term id ever added (commit requires vocab > max_term_id)
    // committed postings; after later adds, removes or a compaction they stay the base of the next commit (has_base), exact
    // for rows [0, committed_rows)
    Postings post;
    bool committed = false, has_base = false;
    int64_t committed_rows = 0;
    int64_t epoch = 0;              // bumped by every change of the rows (add, remove, compact, synth fill)
    CommitPrep prep;                // made by commit_local, used by the commit_global that follows it
    int64_t vocab = 0, n_docs_global = 0, total_len_global = 0;
    std::vector<float> idf;         // [vocab] and avgdl of the last commit: compaction rebuilds the postings with them
    double avgdl = 1.0;
    int64_t ord_base = 0, ord_stride = 1;   // global ordinal of local row r = ord_base + r * ord_stride
    int64_t commit_epoch = -1;      // epoch of the last commit (a redeal needs an index unchanged since then)
    struct RedealSession* redeal = nullptr;   // open krag_redeal_* session: every other call is refused
    bool broken = false;            // a redeal failed after rows had moved: only krag_index_drop is allowed
    ~krag_index();
};

// an open krag_redeal_* session: the plan and the figures krag_last_compact reports
struct RedealSession {
    RedealPlan plan;
    bool prepared = false, moved = false;
    int64_t packed = 0, unpacked = 0, bytes_moved = 0;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ~RedealSession()
    {
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    }
};
krag_index::~krag_index() { delete redeal; }

namespace {

// A search slot for one call.  `st` is the stream the call enqueues its work with the slot's buffers on: the slot's own
// stream (host-buffer searches, which synchronise it before they return) or the caller's (stage API, which returns with
// the work queued).  The lease orders `st` after the slot's previous user and records the slot's `done` event on `st` when
// it ends, so a slot passes to the next call only once the GPU has finished with it.  Buffers that grow (DevArray::reserve)
// synchronise `st` before freeing the old allocation, which therefore also waits for the previous user.
struct SlotLease {
    krag_ctx* c;
    Slot* s;
    cudaStream_t st;
    explicit SlotLease(krag_ctx* ctx) : SlotLease(ctx, nullptr, true) {}
    SlotLease(krag_ctx* ctx, cudaStream_t caller) : SlotLease(ctx, caller, false) {}
    ~SlotLease()
    {
        cudaEventRecord(s->done, st);
        give_back();
    }

private:
    SlotLease(krag_ctx* ctx, cudaStream_t caller, bool own) : c(ctx)
    {
        {
            std::unique_lock<std::mutex> lk(c->mu);
            c->cv.wait(lk, [&] { return !c->free_slots.empty(); });
            s = c->free_slots.back();
            c->free_slots.pop_back();
        }
        st = own ? s->st : caller;
        const cudaError_t e = cudaStreamWaitEvent(st, s->done, 0);
        if (e != cudaSuccess) {
            give_back();
            KRAG_CUDA(e);
        }
    }
    void give_back()
    {
        {
            std::lock_guard<std::mutex> lk(c->mu);
            c->free_slots.push_back(s);
        }
        c->cv.notify_one();
    }
};

// Called by every mutation under the index's unique lock, before it changes anything: blocks until the search work already
// issued has finished.  Stage calls return with their kernels queued on the caller's stream; each recorded its slot's
// `done` event after them, and every later user of a slot is ordered after that event, so the last record of each slot's
// event covers all the work ever issued with the slot.  Work on other indexes of the context is waited for as well.
void wait_issued_searches(const krag_index* ix)
{
    for (const auto& s : ix->ctx->all_slots) KRAG_CUDA(cudaEventSynchronize(s->done));
}

const uint32_t* alive_ptr(const krag_index* ix) { return ix->has_dead ? ix->alive_d.p : nullptr; }
OrdMap ord_map(const krag_index* ix) { return OrdMap{(uint32_t)ix->ord_base, (uint32_t)ix->ord_stride}; }
int64_t ord_last(const krag_index* ix) { return ix->ord_base + (ix->rows.n > 0 ? (ix->rows.n - 1) * ix->ord_stride : 0); }

// every call on an index except the redeal session's own and drop: refused while a session is open or after a failed one
void require_idle(const krag_index* ix)
{
    KRAG_REQUIRE(!ix->broken, KRAG_E_STATE, "index is unusable: a redeal failed after rows had moved (drop it)");
    KRAG_REQUIRE(!ix->redeal, KRAG_E_STATE, "a redeal session is open on this index");
}

void check_P(int P) { KRAG_REQUIRE(P >= 1 && P <= KRAG_MAX_POOL, KRAG_E_INVALID, "candidate pool must be in [1, 1024]"); }

// the slot's staging for the streamed scan of a host-rows index, grown to this call's shape on st, the stream the lease
// ordered after the slot's previous user.  copy_st needs no wait of its own: every copy into a staging buffer waits for a
// `freed` event recorded on st (launch_dense_scan).
ScanStaging scan_staging(const krag_index* ix, Slot* s, int batch, int P, cudaStream_t st)
{
    if (!s->copy_st) {
        KRAG_CUDA(cudaStreamCreateWithFlags(&s->copy_st, cudaStreamNonBlocking));
        for (cudaEvent_t* e : {&s->copied[0], &s->copied[1], &s->freed[0], &s->freed[1]})
            KRAG_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    }
    const int64_t R = stream_scan_chunk_rows(ix->rows.dpad);
    const int64_t half = (R < ix->rows.n ? R : ix->rows.n) * ix->rows.dpad;
    s->stage.reserve(2 * half, 0, st);
    s->fold.reserve(2 * (int64_t)(batch > 256 ? batch : 256) * P, 0, st);
    s->q_sel.reserve((int64_t)256 * ix->rows.dpad, 0, st);
    s->k_sel.reserve((int64_t)256 * P, 0, st);
    return ScanStaging{{s->stage.p, s->stage.p + half}, R, s->copy_st, {s->copied[0], s->copied[1]}, {s->freed[0], s->freed[1]},
                       s->fold.p, s->q_sel.p, s->k_sel.p};
}

// dense candidates for device-resident padded queries: the dense mode's choice of kernel, then K2 or K1
void dense_candidates_dev(krag_index* ix, Slot* s, const float* d_q, int batch, int P, uint64_t* d_keys, cudaStream_t st,
                          const uint32_t* eligible = nullptr)
{
    krag_ctx* c = ix->ctx;
    const DenseRows& r = ix->rows;
    const uint32_t* alive = eligible ? eligible : alive_ptr(ix);     // rows the scan may return (tombstones [& filter])
    if (r.n == 0) {
        KRAG_CUDA(cudaMemsetAsync(d_keys, 0xFF, sizeof(uint64_t) * (size_t)batch * P, st));
        return;
    }
    KRAG_REQUIRE(ord_last(ix) < 0xFFFFFFFFll, KRAG_E_UNSUPPORTED, "global ordinal exceeds 32 bits");
    s->part.reserve((int64_t)dense_scan_part_elems(c->di, P), 0, st);
    const int mode = c->cfg.dense_mode;
    ScanStaging sg{};
    if (r.host()) sg = scan_staging(ix, s, batch, P, st);
    // host rows: K2 whenever it can serve them (K1 streams every row over the host link); device rows: K2 when forced, or
    // for the batches and indexes it serves faster
    const TcOp op = tc_operand(r, mode == KRAG_DENSE_TC_BF16, mode == KRAG_DENSE_TC_TF32);
    const bool use_tc = (r.host() ? mode != KRAG_DENSE_SCAN
                                  : mode == KRAG_DENSE_TC || mode == KRAG_DENSE_TC_TF32 ||
                                        ((mode == KRAG_DENSE_AUTO || mode == KRAG_DENSE_TC_BF16) && dense_tc_wants(r.n, batch))) &&
                        dense_tc_serves(c->di, r, op);
    if (use_tc) {
        const size_t ws = dense_tc_workspace_bytes(c->di, r.n, P, r.host());
        s->tc_ws.reserve((int64_t)ws, 0, st);
        if (launch_dense_tc(c->di, r, op, alive, d_q, batch, P, ord_map(ix), s->tc_ws.p, ws, s->part.p, &sg, d_keys, st)) return;
    }
    KRAG_REQUIRE(r.host() || (mode != KRAG_DENSE_TC && mode != KRAG_DENSE_TC_TF32) || !dense_tc_wants(r.n, 16), KRAG_E_UNSUPPORTED,
                 "tensor-core dense path unavailable for this index/device");
    launch_dense_scan(c->di, r, alive, d_q, batch, P, ord_map(ix), s->part.p, d_keys, st, &sg);
}

void bm25_candidates_dev(krag_index* ix, Slot* s, const uint32_t* d_terms, const int32_t* d_toff, int n_terms_total, int batch,
                         int P, uint64_t* d_keys, cudaStream_t st, const uint32_t* eligible = nullptr)
{
    KRAG_REQUIRE(ix->committed, KRAG_E_STATE, "index has no committed postings (call krag_index_commit)");
    if (n_terms_total < 0) {   // caller did not provide the host copy of the offsets: read the total back (4 bytes)
        int32_t tot = 0;
        KRAG_CUDA(cudaMemcpyAsync(&tot, d_toff + batch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
        n_terms_total = tot;
    }
    s->part.reserve((int64_t)bm25_part_elems(ix->committed_rows, batch, P), 0, st);
    s->bm25_res.reserve((int64_t)bm25_resolve_bytes(ix->committed_rows, n_terms_total), 0, st);
    launch_bm25(ix->ctx->di, ix->post, ix->committed_rows, eligible ? eligible : alive_ptr(ix), d_terms, d_toff, n_terms_total, s->bm25_res.p, batch, P,
                ord_map(ix), s->part.p, d_keys, st);
}

// stage padded queries on the device
const float* upload_queries(krag_index* ix, Slot* s, const float* q, int batch)
{
    const int d = ix->rows.dim, dp = ix->rows.dpad;
    s->q.reserve((int64_t)batch * dp, 0, s->st);
    if (d == dp) {
        KRAG_CUDA(cudaMemcpyAsync(s->q.p, q, sizeof(float) * (size_t)batch * d, cudaMemcpyHostToDevice, s->st));
    } else {
        s->hq.assign((size_t)batch * dp, 0.f);
        for (int b = 0; b < batch; ++b) memcpy(&s->hq[(size_t)b * dp], q + (size_t)b * d, sizeof(float) * d);
        KRAG_CUDA(cudaMemcpyAsync(s->q.p, s->hq.data(), sizeof(float) * (size_t)batch * dp, cudaMemcpyHostToDevice, s->st));
    }
    return s->q.p;
}

void upload_terms(Slot* s, const uint32_t* q_terms, const int32_t* q_toff, int batch)
{
    const int nt = q_toff[batch];
    KRAG_REQUIRE(q_toff[0] == 0 && nt >= 0, KRAG_E_INVALID, "q_term_offsets must start at 0 and be non-decreasing");
    s->terms.reserve(nt > 0 ? nt : 1, 0, s->st);
    s->toff.reserve(batch + 1, 0, s->st);
    if (nt > 0) KRAG_CUDA(cudaMemcpyAsync(s->terms.p, q_terms, sizeof(uint32_t) * (size_t)nt, cudaMemcpyHostToDevice, s->st));
    KRAG_CUDA(cudaMemcpyAsync(s->toff.p, q_toff, sizeof(int32_t) * (size_t)(batch + 1), cudaMemcpyHostToDevice, s->st));
}

void mark_alive(krag_index* ix, int64_t row0, int64_t n, cudaStream_t st)
{
    int64_t words = (ix->rows.n + n + 31) / 32;
    if ((int64_t)ix->alive_h.size() < words) ix->alive_h.resize((size_t)words, 0u);
    for (int64_t r = row0; r < row0 + n; ++r) ix->alive_h[(size_t)(r >> 5)] |= 1u << (r & 31);
    ix->alive_d.reserve(words, (row0 + 31) / 32, st);
    int64_t w0 = row0 >> 5, w1 = (row0 + n + 31) >> 5;
    KRAG_CUDA(cudaMemcpyAsync(ix->alive_d.p + w0, ix->alive_h.data() + w0, sizeof(uint32_t) * (size_t)(w1 - w0),
                              cudaMemcpyHostToDevice, st));
}

// room for the term lists of `rows` rows and nnz entries
void reserve_terms(krag_index* ix, int64_t rows, int64_t nnz, cudaStream_t st)
{
    ix->toff.reserve(rows + 1, ix->rows.n + 1, st);
    ix->dlen.reserve(rows, ix->rows.n, st);
    ix->tid.reserve(nnz > 0 ? nnz : 1, ix->nnz, st);
    ix->ttf.reserve(nnz > 0 ? nnz : 1, ix->nnz, st);
}

// figures of the last commit (krag_last_commit): process-wide, last writer wins
struct CommitReport { float total_ms = 0.f, host_ms = 0.f; int32_t merged = 0; int64_t postings_written = 0, delta_entries = 0; bool valid = false; };
std::mutex g_commit_mu;
CommitReport g_commit;

double ms_since(std::chrono::steady_clock::time_point t0)
{
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// device work both halves of a commit need: the entries to read and, with a base, its survivor counts and the delta's df
void commit_prepare(krag_index* ix, int64_t vocab)
{
    const auto t0 = std::chrono::steady_clock::now();
    cudaStream_t st = ix->ctx->admin;
    CommitPrep& pr = ix->prep;
    pr = CommitPrep{};
    pr.merge = ix->has_base;
    const int64_t row0 = pr.merge ? ix->committed_rows : 0;
    if (row0 > 0) KRAG_CUDA(cudaMemcpyAsync(&pr.e0, ix->toff.p + row0, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    const int64_t n_entries = ix->nnz - pr.e0;
    pr.entry_doc.alloc(n_entries > 0 ? n_entries : 1);
    if (ix->rows.n > row0) launch_expand_entry_doc(ix->toff.p, ix->rows.n - row0, pr.entry_doc.p, st, row0);
    if (pr.merge) {
        count_survivors(ix->post, alive_ptr(ix), vocab, pr.sc, st);
        pr.delta_df.alloc(vocab);
        KRAG_CUDA(cudaMemsetAsync(pr.delta_df.p, 0, sizeof(uint32_t) * (size_t)vocab, st));
        if (n_entries > 0) launch_df_histogram(ix->tid.p + pr.e0, pr.entry_doc.p, alive_ptr(ix), n_entries, pr.delta_df.p, st);
    }
    KRAG_CUDA(cudaStreamSynchronize(st));
    pr.vocab = vocab;
    pr.epoch = ix->epoch;
    pr.valid = true;
    pr.ms = ms_since(t0);
}

void commit_local_impl(krag_index* ix, int64_t vocab, uint32_t* df_out, int64_t* n_live_out, int64_t* total_len_out)
{
    cudaStream_t st = ix->ctx->admin;
    KRAG_REQUIRE(ix->has_sparse || ix->rows.n == 0, KRAG_E_STATE, "index holds no term lists (dense-only)");
    KRAG_REQUIRE(vocab > 0 && vocab < 0x7fffffffll, KRAG_E_INVALID, "vocab out of range");
    // term ids >= vocab would make the df kernel write out of bounds: the largest id is tracked on the host at add time
    KRAG_REQUIRE(ix->nnz == 0 || vocab > (int64_t)ix->max_term_id, KRAG_E_INVALID,
                 "vocab must exceed the largest term id added to the index");
    const auto t0 = std::chrono::steady_clock::now();
    commit_prepare(ix, vocab);
    DevArray<uint32_t> df;
    df.alloc(vocab);
    if (ix->prep.merge) {
        launch_add_u32(ix->prep.sc.per_term.p, ix->prep.delta_df.p, vocab, df.p, st);
    } else {
        KRAG_CUDA(cudaMemsetAsync(df.p, 0, sizeof(uint32_t) * (size_t)vocab, st));
        if (ix->nnz > 0) launch_df_histogram(ix->tid.p, ix->prep.entry_doc.p, alive_ptr(ix), ix->nnz, df.p, st);
    }
    KRAG_CUDA(cudaMemcpyAsync(df_out, df.p, sizeof(uint32_t) * (size_t)vocab, cudaMemcpyDeviceToHost, st));
    live_doc_stats(ix->dlen.p, alive_ptr(ix), ix->rows.n, n_live_out, total_len_out, st);
    ix->prep.ms = ms_since(t0);
}

// idf on the host with glibc log(): the same libm call chain as the reference's math.log.  Split across threads for large
// vocabularies; every value is computed alone, so the bits do not depend on the split.
std::vector<float> host_idf(const uint32_t* df_global, int64_t vocab, int64_t n_docs_global)
{
    std::vector<float> idf((size_t)vocab);
    auto run = [&](int64_t lo, int64_t hi) {
        for (int64_t t = lo; t < hi; ++t) {
            double dfd = (double)df_global[t];
            idf[(size_t)t] = (float)log(1.0 + ((double)n_docs_global - dfd + 0.5) / (dfd + 0.5));
        }
    };
    const int64_t per_thread = (int64_t)1 << 16;
    int64_t n_threads = (vocab + per_thread - 1) / per_thread;
    const int64_t hw = (int64_t)std::thread::hardware_concurrency();
    n_threads = std::min<int64_t>(n_threads, std::min<int64_t>(hw > 0 ? hw : 1, 16));
    if (n_threads <= 1) {
        run(0, vocab);
        return idf;
    }
    std::vector<std::thread> th;
    const int64_t step = (vocab + n_threads - 1) / n_threads;
    for (int64_t i = 0; i < n_threads; ++i) th.emplace_back(run, i * step, std::min(vocab, (i + 1) * step));
    for (auto& t : th) t.join();
    return idf;
}

// the base merged with the rows added since: survivors in base order, then the live new rows, every posting rescored
Postings merge_postings(krag_index* ix, int64_t vocab, const float* idf, double avgdl)
{
    cudaStream_t st = ix->ctx->admin;
    const CommitPrep& pr = ix->prep;
    const int64_t n_entries = ix->nnz - pr.e0;
    DevArray<int64_t> delta_off;
    std::vector<int64_t> h_delta_off;
    df_offsets(pr.delta_df.p, vocab, delta_off, &h_delta_off, st);
    Postings out;
    {
        DevArray<uint32_t> df;
        df.alloc(vocab);
        launch_add_u32(pr.sc.per_term.p, pr.delta_df.p, vocab, df.p, st);
        df_offsets(df.p, vocab, out.off, nullptr, st);
    }
    int64_t nnz = 0;
    KRAG_CUDA(cudaMemcpyAsync(&nnz, out.off.p + vocab, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    out.vocab = vocab;
    out.nnz = nnz;
    out.doc.alloc(nnz > 0 ? nnz : 1);
    out.tf.alloc(nnz > 0 ? nnz : 1);
    out.score.alloc(nnz > 0 ? nnz : 1);
    if (nnz > 0) prepare_tile_index(out.off.p, vocab, ix->rows.n, out, st);
    else empty_tile_index(vocab, ix->rows.n, out);
    write_survivors(ix->post, alive_ptr(ix), pr.sc, out.off.p, nullptr, ix->dlen.p, idf, avgdl, out, st);
    if (n_entries > 0)
        sort_entries_by_term(ix->tid.p + pr.e0, ix->ttf.p + pr.e0, pr.entry_doc.p, alive_ptr(ix), n_entries, vocab, h_delta_off,
                             [&](int64_t q_base, int64_t m, const uint32_t* keys, const uint64_t* vals) {
                                 write_delta(keys, vals, q_base, m, delta_off.p, pr.sc, out.off.p, ix->dlen.p, idf, avgdl, out, st);
                             }, st);
    fill_tile_index(out, st);
    KRAG_CUDA(cudaStreamSynchronize(st));
    return out;
}

void commit_global_impl(krag_index* ix, int64_t vocab, const uint32_t* df_global, int64_t n_docs_global,
                        int64_t total_len_global, int64_t ord_base)
{
    cudaStream_t st = ix->ctx->admin;
    KRAG_REQUIRE(ord_base >= 0 && ord_base + ix->rows.n * ix->ord_stride <= 0xFFFFFFFFll, KRAG_E_UNSUPPORTED, "global ordinal exceeds 32 bits");
    // n_docs_global == 0 is legal: every document deleted (the reference's docstore is then empty and its retriever
    // falls back to vector-only, hybrid_retriever.py:113-121); the postings come out empty and avgdl is irrelevant
    KRAG_REQUIRE(n_docs_global >= 0 && total_len_global >= 0, KRAG_E_INVALID, "n_docs_global / total_len_global must be >= 0");
    KRAG_REQUIRE(ix->nnz == 0 || vocab > (int64_t)ix->max_term_id, KRAG_E_INVALID,
                 "vocab must exceed the largest term id added to the index");
    const auto t0 = std::chrono::steady_clock::now();
    double local_ms = ix->prep.ms;      // commit_local's time; a preparation made here is inside this call's own time
    if (!ix->prep.valid || ix->prep.vocab != vocab || ix->prep.epoch != ix->epoch) {
        commit_prepare(ix, vocab);
        local_ms = 0.0;
    }
    const auto th = std::chrono::steady_clock::now();
    std::vector<float> idf = host_idf(df_global, vocab, n_docs_global);
    const double host_ms = ms_since(th);
    DevArray<float> d_idf;
    d_idf.alloc(vocab);
    KRAG_CUDA(cudaMemcpyAsync(d_idf.p, idf.data(), sizeof(float) * (size_t)vocab, cudaMemcpyHostToDevice, st));
    const double avgdl = n_docs_global > 0 ? (double)total_len_global / (double)n_docs_global : 1.0;
    const bool merged = ix->prep.merge;
    const int64_t delta_entries = ix->nnz - ix->prep.e0;
    if (merged) {
        Postings out = merge_postings(ix, vocab, d_idf.p, avgdl);   // the base stays intact until this has succeeded
        ix->post = std::move(out);
    } else {
        ix->has_base = false;                                         // build_postings writes into ix->post
        ix->committed = false;
        build_postings(ix->tid.p, ix->ttf.p, ix->prep.entry_doc.p, ix->dlen.p, alive_ptr(ix), ix->nnz, vocab, d_idf.p, avgdl,
                       ix->rows.n, ix->post, st);
    }
    KRAG_CUDA(cudaStreamSynchronize(st));
    d_idf.release();
    ix->prep = CommitPrep{};
    ix->idf = std::move(idf);
    ix->avgdl = avgdl;
    ix->vocab = vocab;
    ix->n_docs_global = n_docs_global;
    ix->total_len_global = total_len_global;
    ix->ord_base = ord_base;
    ix->committed = true;
    ix->has_base = true;
    ix->committed_rows = ix->rows.n;
    ix->commit_epoch = ix->epoch;
    CommitReport rep;
    rep.total_ms = (float)(local_ms + ms_since(t0));
    rep.host_ms = (float)host_ms;
    rep.merged = merged ? 1 : 0;
    rep.postings_written = ix->post.nnz;
    rep.delta_entries = delta_entries;
    rep.valid = true;
    std::lock_guard<std::mutex> lk(g_commit_mu);
    g_commit = rep;
}

// figures of the last compaction (krag_last_compact): process-wide, last writer wins
struct CompactReport { float move_ms = 0.f, postings_ms = 0.f; int64_t rows_moved = 0, bytes_moved = 0; bool valid = false; };
std::mutex g_compact_mu;
CompactReport g_compact;

// after a compaction or a redeal has moved the rows: row d holds node ids[d] and every row is alive; exact-size buffers
// where they fit
void renumber_rows(krag_index* ix, std::vector<uint64_t> ids, cudaStream_t st)
{
    const int64_t n = (int64_t)ids.size();
    ix->id2row.clear();
    ix->id2row.reserve((size_t)n);
    for (int64_t d = 0; d < n; ++d) ix->id2row[ids[(size_t)d]] = d;
    ix->node_ids = std::move(ids);
    const int64_t words = (n + 31) / 32;
    ix->alive_h.assign((size_t)words, 0xFFFFFFFFu);
    if (n & 31) ix->alive_h.back() = (1u << (n & 31)) - 1u;
    if (words > 0)
        KRAG_CUDA(cudaMemcpyAsync(ix->alive_d.p, ix->alive_h.data(), sizeof(uint32_t) * (size_t)words, cudaMemcpyHostToDevice, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    ix->n_live = n;
    ix->has_dead = false;
    ix->epoch++;
    ix->prep = CommitPrep{};
    ix->rows.shrink(n, st);
    ix->alive_d.shrink(words > 0 ? words : 1, st);
    if (ix->has_sparse) ix->dlen.shrink(n > 0 ? n : 1, st);
}

// krag_index_compact on an index with dead rows and ordinal stride 1 (writer lock held)
void compact_impl(krag_index* ix)
{
    cudaStream_t st = ix->ctx->admin;
    CompactPlan plan;
    compact_plan(ix->alive_d.p, ix->rows.n, ix->has_sparse ? ix->toff.p : nullptr, plan, st);
    const int64_t n = plan.n_live;
    const int64_t nnz = ix->has_sparse ? plan.h_toff_new[(size_t)n] : 0;
    CompactReport rep;

    // postings first, while the old row numbers and alive bits are still in place: the base's survivors renumbered to their
    // ranks, scores and tf unchanged (the statistics they were computed with do not change), into new arrays -- an
    // allocation failure leaves the index as it was
    Postings remapped;
    const bool keep_base = ix->has_base;
    int64_t base_rows = 0;
    if (keep_base) {
        const auto t0 = std::chrono::steady_clock::now();
        DevArray<uint32_t> rank;
        rank.alloc(ix->rows.n);
        launch_rank_of_rows(plan.src.p, n, rank.p, st);
        SurvivorCounts sc;
        count_survivors(ix->post, alive_ptr(ix), ix->post.vocab, sc, st);
        int64_t pn = 0;
        KRAG_CUDA(cudaMemcpyAsync(&pn, sc.before.p + ix->post.vocab, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
        remapped.vocab = ix->post.vocab;
        remapped.nnz = pn;
        remapped.doc.alloc(pn > 0 ? pn : 1);
        remapped.tf.alloc(pn > 0 ? pn : 1);
        remapped.score.alloc(pn > 0 ? pn : 1);
        write_survivors(ix->post, alive_ptr(ix), sc, sc.before.p, rank.p, nullptr, nullptr, 0.0, remapped, st);
        remapped.off = std::move(sc.before);                        // the remapped offsets are the survivors' exclusive scan
        if (pn > 0) prepare_tile_index(remapped.off.p, remapped.vocab, n, remapped, st);
        else empty_tile_index(remapped.vocab, n, remapped);
        fill_tile_index(remapped, st);
        KRAG_CUDA(cudaStreamSynchronize(st));
        base_rows = (int64_t)(std::lower_bound(plan.h_src.begin(), plan.h_src.end(), (uint32_t)ix->committed_rows) - plan.h_src.begin());
        rep.postings_ms = (float)ms_since(t0);
    }

    cudaEvent_t e0, e1;
    KRAG_CUDA(cudaEventCreate(&e0));
    KRAG_CUDA(cudaEventCreate(&e1));
    KRAG_CUDA(cudaEventRecord(e0, st));
    if (ix->has_sparse) {
        rep.bytes_moved += compact_rows(ix->dlen.p, sizeof(uint32_t), plan, st);
        rep.bytes_moved += compact_terms(ix->tid.p, ix->ttf.p, ix->toff.p, plan, st);
        KRAG_CUDA(cudaMemcpyAsync(ix->toff.p, plan.toff_new.p, sizeof(int64_t) * (size_t)(n + 1), cudaMemcpyDeviceToDevice, st));
    }
    rep.bytes_moved += ix->rows.compact(plan, st);
    KRAG_CUDA(cudaEventRecord(e1, st));
    KRAG_CUDA(cudaEventSynchronize(e1));
    KRAG_CUDA(cudaEventElapsedTime(&rep.move_ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    rep.rows_moved = n - plan.first;

    // host-side state
    std::vector<uint64_t> ids((size_t)n);
    for (int64_t d = 0; d < n; ++d) ids[(size_t)d] = ix->node_ids[plan.h_src[(size_t)d]];
    plan = CompactPlan{};
    ix->nnz = nnz;
    ix->post = std::move(remapped);      // empty without a base
    ix->committed_rows = base_rows;
    renumber_rows(ix, std::move(ids), st);
    if (ix->has_sparse) {
        ix->toff.shrink(n + 1, st);
        ix->tid.shrink(nnz > 0 ? nnz : 1, st);
        ix->ttf.shrink(nnz > 0 ? nnz : 1, st);
    }

    rep.valid = true;
    std::lock_guard<std::mutex> lk(g_compact_mu);
    g_compact = rep;
}

}  // namespace

extern "C" {

int32_t krag_version(void) { return 100; }
const char* krag_last_error(void) { return g_err.c_str(); }

int32_t krag_init(const krag_config* cfg, krag_ctx** out)
{
    return guarded([&] {
        KRAG_REQUIRE(cfg && out, KRAG_E_INVALID, "null argument");
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        KRAG_REQUIRE(e == cudaSuccess && n > 0, KRAG_E_NO_DEVICE,
                     std::string("no CUDA device: ") + cudaGetErrorString(e) + " (libkaito_rag has no CPU fallback)");
        KRAG_REQUIRE(cfg->device_id >= 0 && cfg->device_id < n, KRAG_E_INVALID, "device_id out of range");
        KRAG_REQUIRE(cfg->row_storage == KRAG_ROWS_DEVICE || cfg->row_storage == KRAG_ROWS_HOST, KRAG_E_INVALID,
                     "row_storage must be KRAG_ROWS_DEVICE or KRAG_ROWS_HOST");
        KRAG_CUDA(cudaSetDevice(cfg->device_id));
        cudaDeviceProp p;
        KRAG_CUDA(cudaGetDeviceProperties(&p, cfg->device_id));
        KRAG_REQUIRE(p.major == 9 && p.minor == 0, KRAG_E_NO_DEVICE,
                     std::string("device is sm_") + std::to_string(p.major) + std::to_string(p.minor) +
                         "; libkaito_rag is built for sm_90a only");
        auto c = std::make_unique<krag_ctx>();
        c->cfg = *cfg;
        if (c->cfg.world_size <= 0) c->cfg.world_size = 1;
        c->di.device = cfg->device_id;
        c->di.sm_count = p.multiProcessorCount;
        c->di.cc_major = p.major;
        c->di.cc_minor = p.minor;
        c->di.smem_optin = p.sharedMemPerBlockOptin;
        KRAG_CUDA(cudaStreamCreateWithFlags(&c->admin, cudaStreamNonBlocking));
        int ns = cfg->search_slots > 0 ? cfg->search_slots : 4;
        for (int i = 0; i < ns; ++i) {
            c->all_slots.push_back(std::make_unique<Slot>());
            KRAG_CUDA(cudaStreamCreateWithFlags(&c->all_slots.back()->st, cudaStreamNonBlocking));
            KRAG_CUDA(cudaEventCreateWithFlags(&c->all_slots.back()->done, cudaEventDisableTiming));
            c->free_slots.push_back(c->all_slots.back().get());
        }
        *out = c.release();
    });
}

int32_t krag_shutdown(krag_ctx* c)
{
    return guarded([&] {
        KRAG_REQUIRE(c, KRAG_E_INVALID, "null context");
        cudaSetDevice(c->di.device);
        cudaDeviceSynchronize();
        delete c;
    });
}

int64_t krag_launch_count(krag_ctx*) { return launch_count(); }
int64_t krag_device_bytes(void) { return device_bytes(); }
int64_t krag_host_pinned_bytes(void) { return host_pinned_bytes(); }
void* krag_ctx_stream(krag_ctx* c) { return c ? (void*)c->all_slots[0]->st : nullptr; }

int32_t krag_index_create(krag_ctx* c, const char* name, int32_t dim, krag_index** out)
{
    return guarded([&] {
        KRAG_REQUIRE(c && name && out, KRAG_E_INVALID, "null argument");
        KRAG_REQUIRE(dim >= 1 && dim <= 16384, KRAG_E_INVALID, "dim must be in [1, 16384]");
        krag_index* ix = new krag_index();
        ix->ctx = c;
        ix->name = name;
        ix->rows.init(dim, c->cfg.row_storage == KRAG_ROWS_HOST);
        ix->ord_base = 0;
        *out = ix;
    });
}

int32_t krag_index_drop(krag_index* ix)
{
    return guarded([&] {
        KRAG_REQUIRE(ix, KRAG_E_INVALID, "null index");
        {
            std::unique_lock<std::shared_mutex> lk(ix->mu);
            cudaSetDevice(ix->ctx->di.device);
            cudaDeviceSynchronize();
        }
        delete ix;
    });
}

int32_t krag_index_reserve(krag_index* ix, int64_t rows, int64_t nnz)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && rows >= 0, KRAG_E_INVALID, "bad argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        ix->rows.reserve(rows, ix->ctx->cfg.dense_mode, ix->ctx->admin);
        if (nnz > 0) reserve_terms(ix, rows, nnz, ix->ctx->admin);
    });
}

int32_t krag_index_add(krag_index* ix, int64_t n, const uint64_t* node_ids, const float* vecs,
                       const int64_t* term_offsets, const uint32_t* term_ids, const uint16_t* term_tf,
                       const uint32_t* doc_len)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && n >= 0, KRAG_E_INVALID, "bad argument");
        if (n == 0) return;
        KRAG_REQUIRE(node_ids && vecs, KRAG_E_INVALID, "node_ids and vecs are required");
        const bool sparse = term_offsets != nullptr;
        KRAG_REQUIRE(!sparse || (term_ids && term_tf && doc_len), KRAG_E_INVALID, "term_ids/term_tf/doc_len required with term_offsets");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        cudaStream_t st = ix->ctx->admin;
        KRAG_REQUIRE(ix->rows.n == 0 || sparse == ix->has_sparse, KRAG_E_STATE,
                     "an index is either hybrid (term lists for every node) or dense-only");
        {
            std::unordered_map<uint64_t, int64_t> batch;   // ids must be new to the index AND unique inside the call
            batch.reserve((size_t)n);
            for (int64_t i = 0; i < n; ++i) {
                KRAG_REQUIRE(ix->id2row.find(node_ids[i]) == ix->id2row.end(), KRAG_E_INVALID, "duplicate node id");
                KRAG_REQUIRE(batch.emplace(node_ids[i], i).second, KRAG_E_INVALID, "duplicate node id inside the batch");
            }
        }
        const int64_t add_nnz = sparse ? term_offsets[n] - term_offsets[0] : 0;
        KRAG_REQUIRE(!sparse || (term_offsets[0] == 0 && add_nnz >= 0), KRAG_E_INVALID, "term_offsets must start at 0");
        if (sparse) reserve_terms(ix, ix->rows.n + n, ix->nnz + add_nnz, st);
        ix->rows.append(vecs, n, ix->ctx->cfg.dense_mode, st);   // rows [rows.n, rows.n + n), published below
        std::vector<int64_t> shifted;
        if (sparse) {
            shifted.resize((size_t)n + 1);
            for (int64_t i = 0; i <= n; ++i) {
                KRAG_REQUIRE(i == 0 || term_offsets[i] >= term_offsets[i - 1], KRAG_E_INVALID, "term_offsets must be non-decreasing");
                shifted[(size_t)i] = ix->nnz + term_offsets[i];
            }
            KRAG_CUDA(cudaMemcpyAsync(ix->toff.p + ix->rows.n, shifted.data(), sizeof(int64_t) * (size_t)(n + 1),
                                      cudaMemcpyHostToDevice, st));
            KRAG_CUDA(cudaMemcpyAsync(ix->dlen.p + ix->rows.n, doc_len, sizeof(uint32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
            if (add_nnz > 0) {
                uint32_t mx = ix->max_term_id;
                for (int64_t i = 0; i < add_nnz; ++i) mx = term_ids[i] > mx ? term_ids[i] : mx;
                ix->max_term_id = mx;
                KRAG_CUDA(cudaMemcpyAsync(ix->tid.p + ix->nnz, term_ids, sizeof(uint32_t) * (size_t)add_nnz, cudaMemcpyHostToDevice, st));
                KRAG_CUDA(cudaMemcpyAsync(ix->ttf.p + ix->nnz, term_tf, sizeof(uint16_t) * (size_t)add_nnz, cudaMemcpyHostToDevice, st));
            }
        }
        mark_alive(ix, ix->rows.n, n, st);
        KRAG_CUDA(cudaStreamSynchronize(st));
        for (int64_t i = 0; i < n; ++i) {
            ix->id2row[node_ids[i]] = ix->rows.n + i;
            ix->node_ids.push_back(node_ids[i]);
        }
        ix->rows.n += n;
        ix->n_live += n;
        ix->nnz += add_nnz;
        ix->has_sparse = sparse;
        ix->epoch++;
        ix->committed = false;  // postings are stale until the next commit (reference rebuilds per query)
    });
}

int32_t krag_index_remove(krag_index* ix, int64_t n, const uint64_t* node_ids, int64_t* n_removed)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && (n == 0 || node_ids), KRAG_E_INVALID, "bad argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        int64_t removed = 0;
        for (int64_t i = 0; i < n; ++i) {
            auto it = ix->id2row.find(node_ids[i]);
            if (it == ix->id2row.end()) continue;
            int64_t r = it->second;
            ix->alive_h[(size_t)(r >> 5)] &= ~(1u << (r & 31));
            KRAG_CUDA(cudaMemcpyAsync(ix->alive_d.p + (r >> 5), &ix->alive_h[(size_t)(r >> 5)], sizeof(uint32_t),
                                      cudaMemcpyHostToDevice, ix->ctx->admin));
            ix->id2row.erase(it);
            ++removed;
        }
        KRAG_CUDA(cudaStreamSynchronize(ix->ctx->admin));
        if (removed) { ix->has_dead = true; ix->n_live -= removed; ix->epoch++; }
        if (n_removed) *n_removed = removed;
    });
}

int32_t krag_index_compact(krag_index* ix, int64_t* n_reclaimed_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix, KRAG_E_INVALID, "null index");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        KRAG_REQUIRE(ix->ord_stride == 1, KRAG_E_UNSUPPORTED,
                     "compaction needs ordinal stride 1: rows of a round-robin shard cannot move down without leaving it");
        if (n_reclaimed_out) *n_reclaimed_out = 0;
        if (!ix->has_dead || ix->n_live == ix->rows.n) return;
        const int64_t before = ix->rows.n;
        compact_impl(ix);
        if (n_reclaimed_out) *n_reclaimed_out = before - ix->rows.n;
    });
}

int32_t krag_last_compact(float* move_ms, float* postings_ms, int64_t* rows_moved, int64_t* bytes_moved)
{
    return guarded([&] {
        KRAG_REQUIRE(move_ms && postings_ms && rows_moved && bytes_moved, KRAG_E_INVALID, "null argument");
        std::lock_guard<std::mutex> lk(g_compact_mu);
        KRAG_REQUIRE(g_compact.valid, KRAG_E_STATE, "no compaction has run yet");
        *move_ms = g_compact.move_ms; *postings_ms = g_compact.postings_ms;
        *rows_moved = g_compact.rows_moved; *bytes_moved = g_compact.bytes_moved;
    });
}

// ------------------------------------------------------------- redeal: compaction of round-robin shards together
int32_t krag_index_alive_bitmap(krag_index* ix, uint32_t* out, int64_t cap_words, int64_t* words_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && words_out, KRAG_E_INVALID, "null argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        const int64_t words = (ix->rows.n + 31) / 32;
        *words_out = words;
        if (!out) return;
        KRAG_REQUIRE(cap_words >= words, KRAG_E_INVALID, "bitmap buffer holds fewer words than the index has rows / 32");
        if (words > 0) memcpy(out, ix->alive_h.data(), sizeof(uint32_t) * (size_t)words);
    });
}

static RedealSession* open_session(krag_index* ix)
{
    KRAG_REQUIRE(!ix->broken, KRAG_E_STATE, "index is unusable: a redeal failed after rows had moved (drop it)");
    KRAG_REQUIRE(ix->redeal, KRAG_E_STATE, "no redeal session is open on this index");
    return ix->redeal;
}

static RedealRows redeal_rows(krag_index* ix)
{
    const bool sp = ix->has_sparse;
    return ix->rows.redeal_rows(sp ? ix->dlen.p : nullptr, sp ? ix->toff.p : nullptr, sp ? ix->tid.p : nullptr, sp ? ix->ttf.p : nullptr);
}

int32_t krag_redeal_begin(krag_index* ix, const uint32_t* alive_all, int64_t words, int64_t window_rows, int64_t* n_windows_out,
                          int64_t* n_live_out, int64_t* row_bytes_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && alive_all && n_windows_out && n_live_out && row_bytes_out && words >= 0 && window_rows >= 1,
                     KRAG_E_INVALID, "bad argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        const int G = (int)ix->ord_stride, s = (int)ix->ord_base;
        KRAG_REQUIRE(s < G, KRAG_E_STATE, "not a round-robin shard: the ordinal base must be below the stride");
        KRAG_REQUIRE(words >= (ix->rows.n + 31) / 32, KRAG_E_INVALID, "the bitmaps hold fewer words than this shard has rows / 32");
        KRAG_REQUIRE(ix->committed && ix->commit_epoch == ix->epoch, KRAG_E_STATE,
                     "rows were added or removed since the last commit: commit before the redeal");
        for (int64_t r = 0; r < ix->rows.n; ++r)
            KRAG_REQUIRE(ix->node_ids[(size_t)r] == (uint64_t)(s + r * G), KRAG_E_STATE,
                         "a node id differs from its global ordinal: the redeal renumbers node ids to the new ordinals");
        const uint32_t* own = alive_all + (size_t)s * (size_t)words;
        const int64_t own_words = (ix->rows.n + 31) / 32;
        bool same = own_words == 0 || memcmp(own, ix->alive_h.data(), sizeof(uint32_t) * (size_t)own_words) == 0;
        for (int64_t w = own_words; w < words; ++w) same = same && own[w] == 0;
        KRAG_REQUIRE(same, KRAG_E_INVALID, "this shard's bitmap in alive_all differs from its alive rows");
        // every shard's rows carry a bf16 copy or none: a shard whose copy the dense mode asks for but does not exist yet
        // builds it from its rows here
        ix->rows.reserve(ix->rows.n, ix->ctx->cfg.dense_mode, ix->ctx->admin);
        const bool has_xh = ix->rows.keeps_bf16(ix->ctx->cfg.dense_mode);
        auto sess = std::make_unique<RedealSession>();
        redeal_plan(alive_all, G, s, words, ix->rows.n, ix->has_sparse ? ix->toff.p : nullptr, has_xh, ix->rows.dpad, window_rows, sess->plan,
                    ix->ctx->admin);
        *n_windows_out = sess->plan.n_windows;
        *n_live_out = sess->plan.n_live;
        *row_bytes_out = sess->plan.row_bytes;
        ix->redeal = sess.release();
    });
}

int32_t krag_redeal_tables(krag_index* ix, int64_t* send_rows, int64_t* send_entries, int64_t* recv_rows)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && send_rows && send_entries && recv_rows, KRAG_E_INVALID, "null argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        const RedealPlan& p = open_session(ix)->plan;
        const size_t n = p.send_rows.size();
        std::copy(p.send_rows.begin(), p.send_rows.end(), send_rows);
        std::copy(p.send_ents.begin(), p.send_ents.begin() + n, send_entries);
        std::copy(p.recv_rows.begin(), p.recv_rows.begin() + n, recv_rows);
    });
}

int32_t krag_redeal_prepare(krag_index* ix, const int64_t* recv_entries)
{
    return guarded([&] {
        KRAG_REQUIRE(ix, KRAG_E_INVALID, "null index");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        RedealSession* ss = open_session(ix);
        KRAG_REQUIRE(!ss->prepared, KRAG_E_STATE, "the redeal session is already prepared");
        KRAG_REQUIRE(recv_entries || ss->plan.n_windows == 0, KRAG_E_INVALID, "null argument");
        for (int64_t i = 0; i < ss->plan.n_windows * ss->plan.G; ++i)
            KRAG_REQUIRE(recv_entries[i] >= 0 && (ix->has_sparse || recv_entries[i] == 0), KRAG_E_INVALID, "bad entry count");
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        const bool sp = ix->has_sparse;
        redeal_prepare(recv_entries, sp ? ix->toff.p : nullptr, sp ? ix->tid.p : nullptr, sp ? ix->ttf.p : nullptr, ss->plan,
                       ix->ctx->admin);
        ss->prepared = true;
    });
}

int32_t krag_dev_redeal_pack(krag_index* ix, int64_t window, void* d_rows, void* d_entries, void* stream)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && d_rows && d_entries, KRAG_E_INVALID, "null argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        RedealSession* ss = open_session(ix);
        const RedealPlan& p = ss->plan;
        KRAG_REQUIRE(ss->prepared && window == ss->packed && ss->packed == ss->unpacked && window < p.n_windows, KRAG_E_STATE,
                     "windows are packed in ascending order, each after the previous one was unpacked");
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        cudaStream_t st = (cudaStream_t)stream;
        if (!ss->e0) {
            KRAG_CUDA(cudaEventCreate(&ss->e0));
            KRAG_CUDA(cudaEventCreate(&ss->e1));
            KRAG_CUDA(cudaEventRecord(ss->e0, st));
        }
        redeal_pack(redeal_rows(ix), p, window, d_rows, d_entries, st);
        const size_t a = (size_t)(window * p.G), b = (size_t)((window + 1) * p.G);
        ss->bytes_moved += (p.seg_row[b] - p.seg_row[a]) * p.row_bytes;
        for (size_t i = a; i < b; ++i) ss->bytes_moved += p.send_ents[i] * REDEAL_ENTRY_BYTES;
        ++ss->packed;
    });
}

int32_t krag_dev_redeal_unpack(krag_index* ix, int64_t window, const void* d_rows, const void* d_entries, void* stream)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && d_rows && d_entries, KRAG_E_INVALID, "null argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        RedealSession* ss = open_session(ix);
        KRAG_REQUIRE(window == ss->unpacked && ss->packed == window + 1, KRAG_E_STATE, "unpack the window that was packed last");
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        ss->moved = true;
        redeal_unpack(redeal_rows(ix), ss->plan, window, d_rows, d_entries, (cudaStream_t)stream);
        ++ss->unpacked;
    });
}

int32_t krag_redeal_finish(krag_index* ix, void* stream, int64_t* n_rows_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && n_rows_out, KRAG_E_INVALID, "null argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        RedealSession* ss = open_session(ix);
        RedealPlan& p = ss->plan;
        KRAG_REQUIRE(ss->prepared && ss->unpacked == p.n_windows, KRAG_E_STATE, "windows remain to be moved");
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        ss->moved = true;
        cudaStream_t st = (cudaStream_t)stream, ad = ix->ctx->admin;
        CompactReport rep;
        if (ss->e0) {
            KRAG_CUDA(cudaEventRecord(ss->e1, st));
            KRAG_CUDA(cudaEventSynchronize(ss->e1));
            KRAG_CUDA(cudaEventElapsedTime(&rep.move_ms, ss->e0, ss->e1));
        }
        KRAG_CUDA(cudaStreamSynchronize(st));
        const int64_t n = p.n_new, G = p.G, s = p.s;
        if (ix->has_sparse) {
            ix->toff = std::move(p.toff_new);
            ix->tid = std::move(p.tid_new);
            ix->ttf = std::move(p.ttf_new);
            ix->nnz = p.ent_base.back();
            if (ix->nnz > 0) ix->max_term_id = std::max<uint32_t>(ix->max_term_id, (uint32_t)(ix->vocab - 1));   // every shard's terms are below the committed vocab
        }
        std::vector<uint64_t> ids((size_t)n);
        for (int64_t j = 0; j < n; ++j) ids[(size_t)j] = (uint64_t)(s + j * G);
        ix->post = Postings{};          // no base: the collective commit that follows is a full build under the same statistics
        ix->committed = false;
        ix->has_base = false;
        ix->committed_rows = 0;
        renumber_rows(ix, std::move(ids), ad);
        rep.rows_moved = p.n_send;
        rep.bytes_moved = ss->bytes_moved;
        rep.valid = true;
        delete ss;
        ix->redeal = nullptr;
        *n_rows_out = n;
        std::lock_guard<std::mutex> g(g_compact_mu);
        g_compact = rep;
    });
}

int32_t krag_redeal_abort(krag_index* ix)
{
    return guarded([&] {
        KRAG_REQUIRE(ix, KRAG_E_INVALID, "null index");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        KRAG_REQUIRE(ix->redeal, KRAG_E_STATE, "no redeal session is open on this index");
        cudaSetDevice(ix->ctx->di.device);
        cudaDeviceSynchronize();
        if (ix->redeal->moved) ix->broken = true;
        delete ix->redeal;
        ix->redeal = nullptr;
    });
}

int32_t krag_last_commit(float* total_ms, float* host_ms, int32_t* merged, int64_t* postings_written, int64_t* delta_entries)
{
    return guarded([&] {
        KRAG_REQUIRE(total_ms && host_ms && merged && postings_written && delta_entries, KRAG_E_INVALID, "null argument");
        std::lock_guard<std::mutex> lk(g_commit_mu);
        KRAG_REQUIRE(g_commit.valid, KRAG_E_STATE, "no commit has run yet");
        *total_ms = g_commit.total_ms; *host_ms = g_commit.host_ms; *merged = g_commit.merged;
        *postings_written = g_commit.postings_written; *delta_entries = g_commit.delta_entries;
    });
}

int32_t krag_index_commit_local(krag_index* ix, int64_t vocab, uint32_t* df_out, int64_t* n_live_out, int64_t* total_len_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && df_out && n_live_out && total_len_out, KRAG_E_INVALID, "null argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        commit_local_impl(ix, vocab, df_out, n_live_out, total_len_out);
    });
}

int32_t krag_index_commit_global(krag_index* ix, int64_t vocab, const uint32_t* df_global, int64_t n_docs_global,
                                 int64_t total_len_global, int64_t ordinal_base)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && df_global, KRAG_E_INVALID, "null argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        commit_global_impl(ix, vocab, df_global, n_docs_global, total_len_global, ordinal_base);
    });
}

int32_t krag_index_commit(krag_index* ix, int64_t vocab)
{
    return guarded([&] {
        KRAG_REQUIRE(ix, KRAG_E_INVALID, "null index");
        KRAG_REQUIRE(vocab >= 1 && vocab <= (int64_t)1 << 31, KRAG_E_INVALID, "vocab must be in [1, 2^31]");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        std::vector<uint32_t> df((size_t)vocab);
        int64_t live = 0, total = 0;
        commit_local_impl(ix, vocab, df.data(), &live, &total);
        commit_global_impl(ix, vocab, df.data(), live, total, ix->ord_base);
    });
}

int32_t krag_index_set_ordinal_map(krag_index* ix, int64_t ordinal_base, int64_t ordinal_stride)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && ordinal_base >= 0 && ordinal_stride >= 1 && ordinal_stride <= 64, KRAG_E_INVALID, "bad argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_REQUIRE(ordinal_base + ix->rows.n * ordinal_stride <= 0xFFFFFFFFll, KRAG_E_UNSUPPORTED, "global ordinal exceeds 32 bits");
        ix->ord_base = ordinal_base; ix->ord_stride = ordinal_stride;
    });
}

int32_t krag_index_stats(krag_index* ix, krag_stats_t* out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && out, KRAG_E_INVALID, "null argument");
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        memset(out, 0, sizeof *out);
        out->n_rows = ix->rows.n; out->n_live = ix->n_live; out->nnz = ix->committed ? ix->post.nnz : ix->nnz;
        out->n_docs_global = ix->n_docs_global; out->total_len_global = ix->total_len_global; out->vocab = ix->vocab;
        out->ordinal_base = ix->ord_base; out->dim = ix->rows.dim; out->dim_padded = ix->rows.dpad;
        out->committed = ix->committed && ix->committed_rows == ix->rows.n;
        out->device_bytes = ix->rows.device_bytes() + ix->alive_d.bytes() + ix->toff.bytes() + ix->tid.bytes() + ix->ttf.bytes() +
                            ix->dlen.bytes() + (ix->committed ? (int64_t)(ix->post.nnz * 10 + (ix->post.vocab + 1) * 8) : 0);
    });
}

int32_t krag_index_node_ids(krag_index* ix, int64_t n, const int64_t* ordinals, uint64_t* out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && (n == 0 || (ordinals && out)), KRAG_E_INVALID, "null argument");
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        for (int64_t i = 0; i < n; ++i) {
            const int64_t off = ordinals[i] - ix->ord_base;
            KRAG_REQUIRE(off >= 0 && off % ix->ord_stride == 0, KRAG_E_NOT_FOUND, "ordinal is not held by this shard");
            const int64_t r = off / ix->ord_stride;
            KRAG_REQUIRE(r < ix->rows.n, KRAG_E_NOT_FOUND, "ordinal is not held by this shard");
            out[i] = ix->node_ids[(size_t)r];
        }
    });
}

// ------------------------------------------------------------------ host-buffer search
int32_t krag_search_dense(krag_index* ix, int32_t batch, const float* q, int32_t k, float* out_l2sq, int64_t* out_ord)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && q && out_l2sq && out_ord && batch >= 1, KRAG_E_INVALID, "bad argument");
        check_P(k);
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        SlotLease lease(ix->ctx);
        Slot* s = lease.s;
        const float* dq = upload_queries(ix, s, q, batch);
        s->dense_keys.reserve((int64_t)batch * k, 0, s->st);
        dense_candidates_dev(ix, s, dq, batch, k, s->dense_keys.p, s->st);
        std::vector<uint64_t> keys((size_t)batch * k);
        KRAG_CUDA(cudaMemcpyAsync(keys.data(), s->dense_keys.p, sizeof(uint64_t) * keys.size(), cudaMemcpyDeviceToHost, s->st));
        KRAG_CUDA(cudaStreamSynchronize(s->st));
        for (size_t i = 0; i < keys.size(); ++i) {
            if (keys[i] == KEY_PAD) { out_l2sq[i] = INFINITY; out_ord[i] = -1; }
            else { out_l2sq[i] = key_value_asc(keys[i]); out_ord[i] = (int64_t)key_ordinal(keys[i]); }
        }
    });
}

int32_t krag_search_bm25(krag_index* ix, int32_t batch, const uint32_t* q_terms, const int32_t* q_toff, int32_t k,
                         float* out_score, int64_t* out_ord)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && q_toff && out_score && out_ord && batch >= 1, KRAG_E_INVALID, "bad argument");
        check_P(k);
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        SlotLease lease(ix->ctx);
        Slot* s = lease.s;
        upload_terms(s, q_terms, q_toff, batch);
        s->bm25_keys.reserve((int64_t)batch * k, 0, s->st);
        bm25_candidates_dev(ix, s, s->terms.p, s->toff.p, q_toff[batch], batch, k, s->bm25_keys.p, s->st);
        std::vector<uint64_t> keys((size_t)batch * k);
        KRAG_CUDA(cudaMemcpyAsync(keys.data(), s->bm25_keys.p, sizeof(uint64_t) * keys.size(), cudaMemcpyDeviceToHost, s->st));
        KRAG_CUDA(cudaStreamSynchronize(s->st));
        for (size_t i = 0; i < keys.size(); ++i) {
            if (keys[i] == KEY_PAD) { out_score[i] = 0.f; out_ord[i] = -1; }
            else { out_score[i] = key_value_desc(keys[i]); out_ord[i] = (int64_t)key_ordinal(keys[i]); }
        }
    });
}

int32_t krag_retrieve(krag_index* ix, int32_t batch, const float* q, const uint32_t* q_terms, const int32_t* q_toff,
                      int32_t k, double cand_mult, double vector_weight, double text_weight, int32_t fusion_mode,
                      const uint32_t* keyword_allow_bitmap, int64_t keyword_allow_words, double* out_final, float* out_dense,
                      float* out_sparse, int32_t* out_rank, int64_t* out_ord, int32_t* out_count)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && q && out_final && out_dense && out_sparse && out_rank && out_ord && out_count && batch >= 1,
                     KRAG_E_INVALID, "bad argument");
        KRAG_REQUIRE(k >= 1 && k <= KRAG_MAX_TOP_K, KRAG_E_INVALID, "k must be in [1, 300]");
        KRAG_REQUIRE(vector_weight + text_weight > 0, KRAG_E_INVALID, "weights must sum to a positive value");
        // HybridRetriever.__init__ (hybrid_retriever.py:91-98)
        const double total = vector_weight + text_weight;
        const double w_v = vector_weight / total, w_t = text_weight / total;
        const double mult = cand_mult > 1.0 ? cand_mult : 1.0;
        const int P = (int)((double)k * mult);
        check_P(P);
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        // the bitmap is read (n_rows + 31) / 32 words deep: the caller states how many it holds, so a bitmap built
        // before a concurrent krag_index_add is refused instead of over-read
        KRAG_REQUIRE(keyword_allow_bitmap == nullptr || keyword_allow_words >= (ix->rows.n + 31) / 32, KRAG_E_INVALID,
                     "keyword_allow_bitmap holds fewer words than the index has rows / 32");
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        SlotLease lease(ix->ctx);
        Slot* s = lease.s;
        cudaStream_t st = s->st;
        const bool hybrid = q_terms != nullptr && q_toff != nullptr && ix->committed;
        const bool pushdown = (fusion_mode & KRAG_FILTER_PUSHDOWN) != 0 && keyword_allow_bitmap != nullptr;
        fusion_mode &= 0xFF;
        const uint32_t* eligible = nullptr;
        if (pushdown) {   // eligible = allow & alive, consumed by K1/K2/K3 in place of the tombstone bitmap
            const int64_t words = (ix->rows.n + 31) / 32;
            s->allow.reserve(words > 0 ? words : 1, 0, st);
            KRAG_CUDA(cudaMemcpyAsync(s->allow.p, keyword_allow_bitmap, sizeof(uint32_t) * (size_t)words, cudaMemcpyHostToDevice, st));
            if (ix->has_dead && words > 0) launch_bitmap_and(s->allow.p, ix->alive_d.p, words, st);
            eligible = s->allow.p;
        }
        const float* dq = upload_queries(ix, s, q, batch);
        s->dense_keys.reserve((int64_t)batch * P, 0, st);
        dense_candidates_dev(ix, s, dq, batch, P, s->dense_keys.p, st, eligible);
        const uint32_t* d_allow = nullptr;
        if (hybrid) {
            upload_terms(s, q_terms, q_toff, batch);
            s->bm25_keys.reserve((int64_t)batch * P, 0, st);
            bm25_candidates_dev(ix, s, s->terms.p, s->toff.p, q_toff[batch], batch, P, s->bm25_keys.p, st, eligible);
            if (keyword_allow_bitmap && !pushdown) {
                // bitmap is over local rows; fuse tests global ordinals -> shift by ord_base words is only
                // valid when ord_base % 32 == 0; the host path is single-shard (ord_base == 0)
                KRAG_REQUIRE(ix->ord_base == 0 && ix->ord_stride == 1, KRAG_E_UNSUPPORTED, "keyword filter on host path requires ordinal_base 0, stride 1");
                int64_t words = (ix->rows.n + 31) / 32;
                s->allow.reserve(words, 0, st);
                KRAG_CUDA(cudaMemcpyAsync(s->allow.p, keyword_allow_bitmap, sizeof(uint32_t) * (size_t)words, cudaMemcpyHostToDevice, st));
                d_allow = s->allow.p;
            }
        }
        const int64_t nk = (int64_t)batch * k;
        s->out_final.reserve(nk, 0, st); s->out_dense.reserve(nk, 0, st); s->out_sparse.reserve(nk, 0, st);
        s->out_rank.reserve(nk, 0, st); s->out_ord.reserve(nk, 0, st); s->out_count.reserve(batch, 0, st);
        launch_fuse(batch, P, k, s->dense_keys.p, hybrid ? s->bm25_keys.p : nullptr, w_v, w_t, fusion_mode, d_allow,
                    s->out_final.p, s->out_dense.p, s->out_sparse.p, s->out_rank.p, s->out_ord.p, s->out_count.p, st);
        KRAG_CUDA(cudaMemcpyAsync(out_final, s->out_final.p, sizeof(double) * (size_t)nk, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaMemcpyAsync(out_dense, s->out_dense.p, sizeof(float) * (size_t)nk, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaMemcpyAsync(out_sparse, s->out_sparse.p, sizeof(float) * (size_t)nk, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaMemcpyAsync(out_rank, s->out_rank.p, sizeof(int32_t) * (size_t)nk, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaMemcpyAsync(out_ord, s->out_ord.p, sizeof(int64_t) * (size_t)nk, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaMemcpyAsync(out_count, s->out_count.p, sizeof(int32_t) * (size_t)batch, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
    });
}

// ---------------------------------------------------------------- device stage API
int32_t krag_dev_dense_candidates(krag_index* ix, int32_t batch, const float* d_q, int32_t P, uint64_t* d_keys, void* stream)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && d_q && d_keys && batch >= 1, KRAG_E_INVALID, "bad argument");
        check_P(P);
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        SlotLease lease(ix->ctx, (cudaStream_t)stream);
        dense_candidates_dev(ix, lease.s, d_q, batch, P, d_keys, lease.st);
    });
}

int32_t krag_dev_bm25_candidates(krag_index* ix, int32_t batch, const uint32_t* d_terms, const int32_t* d_toff,
                                 const int32_t* h_toff, int32_t P, uint64_t* d_keys, void* stream)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && d_toff && d_keys && batch >= 1, KRAG_E_INVALID, "bad argument");
        check_P(P);
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        SlotLease lease(ix->ctx, (cudaStream_t)stream);
        bm25_candidates_dev(ix, lease.s, d_terms, d_toff, h_toff ? h_toff[batch] : -1, batch, P, d_keys, lease.st);
    });
}

int32_t krag_dev_merge(krag_ctx* c, int32_t n_lists, int32_t batch, int32_t P, const uint64_t* d_in, uint64_t* d_out, void* stream)
{
    return guarded([&] {
        KRAG_REQUIRE(c && d_in && d_out && n_lists >= 1 && batch >= 1, KRAG_E_INVALID, "bad argument");
        check_P(P);
        KRAG_CUDA(cudaSetDevice(c->di.device));
        launch_merge(d_in, n_lists, P, batch, P, (int64_t)batch * P, P, d_out, (cudaStream_t)stream);
    });
}

int32_t krag_dev_fuse(krag_ctx* c, int32_t batch, int32_t P, int32_t k, const uint64_t* d_dense, const uint64_t* d_bm25,
                      double vector_weight, double text_weight, int32_t fusion_mode, const uint32_t* d_allow,
                      double* d_final, float* d_dense_out, float* d_sparse_out, int32_t* d_rank, int64_t* d_ord,
                      int32_t* d_count, void* stream)
{
    return guarded([&] {
        KRAG_REQUIRE(c && d_dense && d_final && d_dense_out && d_sparse_out && d_rank && d_ord && d_count && batch >= 1,
                     KRAG_E_INVALID, "bad argument");
        KRAG_REQUIRE(k >= 1 && k <= KRAG_MAX_POOL, KRAG_E_INVALID, "k out of range");
        check_P(P);
        const double total = vector_weight + text_weight;
        KRAG_REQUIRE(total > 0, KRAG_E_INVALID, "weights must sum to a positive value");
        KRAG_CUDA(cudaSetDevice(c->di.device));
        launch_fuse(batch, P, k, d_dense, d_bm25, vector_weight / total, text_weight / total, fusion_mode, d_allow, d_final,
                    d_dense_out, d_sparse_out, d_rank, d_ord, d_count, (cudaStream_t)stream);
    });
}

// -------------------------------------------------------------------- synthetic / io
int32_t krag_synth_fill(krag_index* ix, int64_t n, int64_t row_base, uint64_t seed, int64_t vocab)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && n >= 0, KRAG_E_INVALID, "bad argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        cudaStream_t st = ix->ctx->admin;
        KRAG_REQUIRE(ix->rows.n == 0, KRAG_E_STATE, "synthetic fill needs an empty index");
        ix->rows.synth(n, row_base, seed, ix->ctx->cfg.dense_mode, st);
        if (vocab > 0) {
            DevArray<int64_t> off; DevArray<uint32_t> ids; DevArray<uint16_t> tf; DevArray<uint32_t> dl; int64_t nnz = 0;
            synth_sparse(n, row_base, seed, vocab, off, ids, tf, dl, &nnz, st);
            ix->toff = std::move(off); ix->tid = std::move(ids); ix->ttf = std::move(tf); ix->dlen = std::move(dl);
            ix->nnz = nnz;
            ix->max_term_id = (uint32_t)(vocab - 1);     // the generator draws ids in [0, vocab)
            ix->has_sparse = true;
        }
        mark_alive(ix, 0, n, st);
        KRAG_CUDA(cudaStreamSynchronize(st));
        ix->node_ids.resize((size_t)n);
        for (int64_t i = 0; i < n; ++i) { ix->node_ids[(size_t)i] = (uint64_t)(row_base + i); ix->id2row[(uint64_t)(row_base + i)] = i; }
        ix->rows.n = n; ix->n_live = n; ix->ord_base = row_base; ix->ord_stride = 1; ix->committed = false;
        ix->has_base = false; ix->post = Postings{}; ix->epoch++;
    });
}

int32_t krag_index_read_rows(krag_index* ix, int64_t row0, int64_t n, float* out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && out && row0 >= 0 && n >= 0 && row0 + n <= ix->rows.n, KRAG_E_INVALID, "row range out of bounds");
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        ix->rows.read(row0, n, out);
    });
}

int32_t krag_debug_read_stored_rows(krag_index* ix, int64_t row0, int64_t n, float* out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && out && row0 >= 0 && n >= 0 && row0 + n <= ix->rows.n, KRAG_E_INVALID, "row range out of bounds");
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        KRAG_REQUIRE(!ix->rows.host(), KRAG_E_UNSUPPORTED, "the stored layout is that of device-resident rows");
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        ix->rows.read_stored(row0, n, out);
    });
}

int32_t krag_index_read_postings(krag_index* ix, uint32_t term, int64_t cap, uint32_t* docs_out, float* scores_out, int64_t* n_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && n_out, KRAG_E_INVALID, "null argument");
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        KRAG_REQUIRE(ix->committed, KRAG_E_STATE, "index not committed");
        KRAG_REQUIRE((int64_t)term < ix->post.vocab, KRAG_E_INVALID, "term id out of range");
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        int64_t be[2];
        KRAG_CUDA(cudaMemcpy(be, ix->post.off.p + term, sizeof be, cudaMemcpyDeviceToHost));
        int64_t cnt = be[1] - be[0];
        *n_out = cnt;
        int64_t m = cnt < cap ? cnt : cap;
        if (m > 0 && docs_out) KRAG_CUDA(cudaMemcpy(docs_out, ix->post.doc.p + be[0], sizeof(uint32_t) * (size_t)m, cudaMemcpyDeviceToHost));
        if (m > 0 && scores_out) KRAG_CUDA(cudaMemcpy(scores_out, ix->post.score.p + be[0], sizeof(float) * (size_t)m, cudaMemcpyDeviceToHost));
    });
}

int32_t krag_index_set_dense_mode(krag_index* ix, int32_t dense_mode, int32_t release_shadow)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && dense_mode >= KRAG_DENSE_AUTO && dense_mode <= KRAG_DENSE_TC_TF32, KRAG_E_INVALID, "bad argument");
        std::unique_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        cudaStream_t st = ix->ctx->admin;
        ix->rows.set_shadow(ix->rows.keeps_bf16(dense_mode, release_shadow != 0), st);
        KRAG_CUDA(cudaStreamSynchronize(st));
        ix->ctx->cfg.dense_mode = dense_mode;
    });
}

int64_t krag_tc_fallback_queries(void) { return dense_tc_fallback_queries(); }
int64_t krag_host_rows_fetched(void) { return host_rows_fetched(); }

int32_t krag_last_dense_kernel(float* ms, int32_t* kernel_id, int64_t* algorithmic_bytes, int64_t* flops)
{
    return guarded([&] {
        KRAG_REQUIRE(ms && kernel_id && algorithmic_bytes && flops, KRAG_E_INVALID, "null argument");
        int kid = 0;
        KRAG_REQUIRE(dense_timer_read(ms, &kid, algorithmic_bytes, flops), KRAG_E_STATE, "no dense kernel timed yet");
        *kernel_id = kid;
    });
}

namespace {
// the prune operand of pass KRAG_TC_PASS_* on the index's rows, for the test hooks (krag_debug_tc_dump_pass, krag_debug_tc_prune)
static_assert(TC_OP_BF16_SPLIT == KRAG_TC_PASS_BF16_SPLIT + 1 && TC_OP_BF16_SHADOW == KRAG_TC_PASS_BF16_SHADOW + 1 &&
                  TC_OP_BF16_HOST == KRAG_TC_PASS_BF16_HOST + 1, "prune passes");
TcOp require_tc_pass(const krag_index* ix, int32_t pass)
{
    const DenseRows& r = ix->rows;
    KRAG_REQUIRE(pass >= KRAG_TC_PASS_TF32 && pass <= KRAG_TC_PASS_BF16_HOST, KRAG_E_INVALID, "unknown prune pass");
    KRAG_REQUIRE(r.n > 0, KRAG_E_STATE, "index has no rows");
    const TcOp op = pass == KRAG_TC_PASS_TF32 ? (r.split() ? TC_OP_TF32S : TC_OP_TF32) : (TcOp)(pass + 1);
    KRAG_REQUIRE(r.host() == (op == TC_OP_BF16_HOST), KRAG_E_UNSUPPORTED,
                 r.host() ? "this prune pass needs device-resident rows" : "the host-rows pass needs a KRAG_ROWS_HOST index");
    KRAG_REQUIRE(op != TC_OP_BF16_SPLIT || r.split(), KRAG_E_UNSUPPORTED, "the index does not keep split rows");
    KRAG_REQUIRE(op != TC_OP_BF16_SHADOW || r.bf16(), KRAG_E_STATE, "the index has no bf16 shadow");
    KRAG_REQUIRE(dense_tc_supported(ix->ctx->di, r.dpad), KRAG_E_UNSUPPORTED, "tensor-core path unavailable");
    return op;
}
}  // namespace

int32_t krag_debug_tc_dump_pass(krag_index* ix, int32_t pass, int32_t nq, const float* q, float* out, int64_t out_elems,
                                int64_t* S_out, int32_t* nq_pad_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && q && S_out && nq_pad_out && nq >= 1 && nq <= 256, KRAG_E_INVALID, "bad argument");
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        const TcOp op = require_tc_pass(ix, pass);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        SlotLease lease(ix->ctx);
        Slot* s = lease.s;
        int64_t S = 0; int nqp = 0;
        const size_t ws = dense_tc_debug_carve(nullptr, nullptr, ix->rows.n, ix->rows.dpad, nq, 0, &S, &nqp);
        *S_out = S; *nq_pad_out = nqp;
        if (!out) return;
        KRAG_REQUIRE(out_elems >= S * nqp, KRAG_E_INVALID, "output buffer too small");
        const float* dq = upload_queries(ix, s, q, nq);
        s->tc_ws.reserve((int64_t)ws, 0, s->st);
        TcDebugWs w;
        dense_tc_debug_carve(&w, s->tc_ws.p, ix->rows.n, ix->rows.dpad, nq, 0, &S, &nqp);
        KRAG_REQUIRE(dense_tc_debug_pass(ix->ctx->di, ix->rows, op, nullptr, dq, nq, w, 0, s->st),
                     KRAG_E_UNSUPPORTED, "tensor-core dump failed");
        KRAG_CUDA(cudaMemcpyAsync(out, w.dump, sizeof(float) * (size_t)(S * nqp), cudaMemcpyDeviceToHost, s->st));
        KRAG_CUDA(cudaStreamSynchronize(s->st));
    });
}

int32_t krag_debug_tc_dump(krag_index* ix, int32_t nq, const float* q, float* out, int64_t out_elems, int64_t* S_out, int32_t* nq_pad_out)
{
    return krag_debug_tc_dump_pass(ix, KRAG_TC_PASS_TF32, nq, q, out, out_elems, S_out, nq_pad_out);
}

int32_t krag_debug_tc_prune(krag_index* ix, int32_t pass, int32_t nq, const float* q, const float* thr, int32_t cap,
                            uint32_t* counts_out, uint32_t* rows_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && q && thr && counts_out && rows_out && nq >= 1 && nq <= 256 && cap >= 1, KRAG_E_INVALID, "bad argument");
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        const TcOp op = require_tc_pass(ix, pass);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        SlotLease lease(ix->ctx);
        Slot* s = lease.s;
        int64_t S = 0; int nqp = 0;
        const size_t ws = dense_tc_debug_carve(nullptr, nullptr, ix->rows.n, ix->rows.dpad, nq, cap, &S, &nqp);
        const float* dq = upload_queries(ix, s, q, nq);
        s->tc_ws.reserve((int64_t)ws, 0, s->st);
        TcDebugWs w;
        dense_tc_debug_carve(&w, s->tc_ws.p, ix->rows.n, ix->rows.dpad, nq, cap, &S, &nqp);
        KRAG_CUDA(cudaMemcpyAsync(w.thr, thr, sizeof(float) * (size_t)nqp, cudaMemcpyHostToDevice, s->st));
        KRAG_REQUIRE(dense_tc_debug_pass(ix->ctx->di, ix->rows, op, alive_ptr(ix), dq, nq, w, cap, s->st),
                     KRAG_E_UNSUPPORTED, "tensor-core prune pass failed");
        KRAG_CUDA(cudaMemcpyAsync(counts_out, w.cand_count, sizeof(uint32_t) * (size_t)nqp, cudaMemcpyDeviceToHost, s->st));
        KRAG_CUDA(cudaMemcpyAsync(rows_out, w.cand_rows, sizeof(uint32_t) * (size_t)nqp * cap, cudaMemcpyDeviceToHost, s->st));
        KRAG_CUDA(cudaStreamSynchronize(s->st));
    });
}

// ------------------------------------------------------------- peer-memory exchange (one process per GPU)
struct krag_p2p {
    krag_ctx* ctx; int rank, world, nl, max_batch, max_P; int64_t slot_words;
    DevArray<uint64_t> own;                  // this rank's mailbox (IPC-exported)
    std::vector<uint64_t*> peers;            // [world] device pointers: own + IPC-opened peers
    DevArray<uint64_t*> d_peers;             // device copy of the pointer table
    unsigned long long seq = 0;
};

int32_t krag_p2p_create(krag_ctx* c, int32_t rank, int32_t world, int32_t max_batch, int32_t max_P, krag_p2p** out, uint8_t* handle_out /*[64]*/)
{
    return guarded([&] {
        KRAG_REQUIRE(c && out && handle_out && world >= 1 && world <= 64 && rank >= 0 && rank < world, KRAG_E_INVALID, "bad argument");
        KRAG_CUDA(cudaSetDevice(c->di.device));
        auto p = std::make_unique<krag_p2p>();
        p->ctx = c; p->rank = rank; p->world = world; p->nl = 2; p->max_batch = max_batch; p->max_P = max_P;
        p->slot_words = (int64_t)2 * max_batch * max_P;
        const size_t words = p2p_mailbox_words(world, 2, max_batch, max_P);
        p->own.alloc((int64_t)words);
        KRAG_CUDA(cudaMemset(p->own.p, 0, words * 8));
        cudaIpcMemHandle_t h;
        KRAG_CUDA(cudaIpcGetMemHandle(&h, p->own.p));
        static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
        memcpy(handle_out, &h, 64);
        p->peers.assign((size_t)world, nullptr);
        p->peers[(size_t)rank] = p->own.p;
        *out = p.release();
    });
}

int32_t krag_p2p_connect(krag_p2p* p, const uint8_t* handles /*[world][64]*/)
{
    return guarded([&] {
        KRAG_REQUIRE(p && handles, KRAG_E_INVALID, "null argument");
        KRAG_CUDA(cudaSetDevice(p->ctx->di.device));
        for (int r = 0; r < p->world; ++r) {
            if (r == p->rank) continue;
            cudaIpcMemHandle_t h;
            memcpy(&h, handles + (size_t)r * 64, 64);
            void* ptr = nullptr;
            KRAG_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
            p->peers[(size_t)r] = (uint64_t*)ptr;
        }
        p->d_peers.alloc(p->world);
        KRAG_CUDA(cudaMemcpy(p->d_peers.p, p->peers.data(), sizeof(uint64_t*) * (size_t)p->world, cudaMemcpyHostToDevice));
    });
}

int32_t krag_dev_exchange_merge(krag_p2p* p, int32_t n_lists, int32_t batch, int32_t P, const uint64_t* d_local, uint64_t* d_merged, void* stream)
{
    return guarded([&] {
        KRAG_REQUIRE(p && p->d_peers.p && d_local && d_merged, KRAG_E_INVALID, "bad argument / not connected");
        KRAG_REQUIRE(n_lists >= 1 && n_lists <= 2 && batch >= 1 && (int64_t)n_lists * batch * P <= p->slot_words, KRAG_E_INVALID,
                     "exchange exceeds the mailbox the ranks agreed on");
        check_P(P);
        KRAG_CUDA(cudaSetDevice(p->ctx->di.device));
        ++p->seq;
        launch_p2p_exchange_merge(p->d_peers.p, p->own.p, p->rank, p->world, p->slot_words, p->seq, n_lists, batch, P, d_local, d_merged,
                                  (cudaStream_t)stream);
    });
}

int32_t krag_p2p_destroy(krag_p2p* p)
{
    return guarded([&] {
        KRAG_REQUIRE(p, KRAG_E_INVALID, "null argument");
        cudaSetDevice(p->ctx->di.device);
        cudaDeviceSynchronize();
        for (int r = 0; r < p->world; ++r) if (r != p->rank && p->peers[(size_t)r]) cudaIpcCloseMemHandle(p->peers[(size_t)r]);
        delete p;
    });
}

// ---------------------------------------------------------------------- K5 embedder
struct krag_embedder { krag_ctx* ctx; Embedder* e; };

int32_t krag_embedder_create(krag_ctx* c, const krag_bert_config* cfg, krag_embedder** out)
{
    return guarded([&] {
        KRAG_REQUIRE(c && cfg && out, KRAG_E_INVALID, "null argument");
        KRAG_CUDA(cudaSetDevice(c->di.device));
        BertConfig bc{cfg->layers, cfg->hidden, cfg->heads, cfg->intermediate, cfg->vocab, cfg->max_position, cfg->type_vocab, cfg->ln_eps};
        krag_embedder* h = new krag_embedder{c, embedder_create(c->di, bc)};
        *out = h;
    });
}
int32_t krag_embedder_load_tensor(krag_embedder* h, const char* name, const float* data, int64_t n)
{
    return guarded([&] {
        KRAG_REQUIRE(h && name && data && n > 0, KRAG_E_INVALID, "bad argument");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        embedder_load(h->e, name, data, n);
    });
}
int32_t krag_embedder_finalize(krag_embedder* h)
{
    return guarded([&] {
        KRAG_REQUIRE(h, KRAG_E_INVALID, "null embedder");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        embedder_finalize(h->e);
    });
}
int32_t krag_embed(krag_embedder* h, int32_t batch, const int32_t* tok_ids, const int32_t* tok_offsets, float* out)
{
    return guarded([&] {
        KRAG_REQUIRE(h && tok_ids && tok_offsets && out && batch >= 1, KRAG_E_INVALID, "bad argument");
        KRAG_REQUIRE(tok_offsets[0] == 0, KRAG_E_INVALID, "tok_offsets must start at 0");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        embedder_forward(h->e, batch, tok_ids, tok_offsets, out);
    });
}
int32_t krag_embed_dev(krag_embedder* h, int32_t batch, const int32_t* tok_ids, const int32_t* tok_offsets, float* d_out,
                       int32_t ld_out, void* stream)
{
    return guarded([&] {
        KRAG_REQUIRE(h && tok_ids && tok_offsets && d_out && batch >= 1 && ld_out >= embedder_hidden(h->e), KRAG_E_INVALID, "bad argument");
        KRAG_REQUIRE(tok_offsets[0] == 0, KRAG_E_INVALID, "tok_offsets must start at 0");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        embedder_forward(h->e, batch, tok_ids, tok_offsets, nullptr, d_out, ld_out, (cudaStream_t)stream);
    });
}
static_assert(KRAG_POOL_CLS == EMB_POOL_CLS && KRAG_POOL_MEAN == EMB_POOL_MEAN, "pooling modes");
int32_t krag_embedder_set_pooling(krag_embedder* h, int32_t mode)
{
    return guarded([&] {
        KRAG_REQUIRE(h, KRAG_E_INVALID, "null embedder");
        KRAG_REQUIRE(mode == KRAG_POOL_CLS || mode == KRAG_POOL_MEAN, KRAG_E_INVALID, "pooling mode must be KRAG_POOL_CLS or KRAG_POOL_MEAN");
        embedder_set_pooling(h->e, mode);
    });
}
static_assert(KRAG_PRECISION_FP32 == EMB_PREC_FP32 && KRAG_PRECISION_FP16 == EMB_PREC_FP16, "precision modes");
int32_t krag_embedder_set_precision(krag_embedder* h, int32_t mode)
{
    return guarded([&] {
        KRAG_REQUIRE(h, KRAG_E_INVALID, "null embedder");
        KRAG_REQUIRE(mode == KRAG_PRECISION_FP32 || mode == KRAG_PRECISION_FP16, KRAG_E_INVALID,
                     "precision must be KRAG_PRECISION_FP32 or KRAG_PRECISION_FP16");
        embedder_set_precision(h->e, mode);
    });
}
int32_t krag_embedder_set_position_offset(krag_embedder* h, int32_t off)
{
    return guarded([&] {
        KRAG_REQUIRE(h, KRAG_E_INVALID, "null embedder");
        KRAG_REQUIRE(off >= 0, KRAG_E_INVALID, "position offset must be >= 0");
        embedder_set_position_offset(h->e, off);
    });
}
int32_t krag_debug_relative_bucket(int32_t rel) { return relative_bucket(rel); }
int32_t krag_embedder_set_rotary(krag_embedder* h, float base)
{
    return guarded([&] {
        KRAG_REQUIRE(h, KRAG_E_INVALID, "null embedder");
        embedder_set_rotary(h->e, base);
    });
}
int32_t krag_debug_rotary_cos_sin(float base, int32_t dh, int32_t pos, float* cos_out, float* sin_out)
{
    return guarded([&] {
        KRAG_REQUIRE(cos_out && sin_out && base > 0.f && dh >= 2 && dh % 2 == 0 && pos >= 0, KRAG_E_INVALID, "bad argument");
        rotary_cos_sin(base, dh, pos, cos_out, sin_out);
    });
}
int32_t krag_debug_embedder_cls_rows(krag_embedder* h, int32_t on)
{
    return guarded([&] {
        KRAG_REQUIRE(h, KRAG_E_INVALID, "null embedder");
        embedder_set_cls_rows_only(h->e, on != 0);
    });
}
static_assert(KRAG_RERANK_SIGMOID == EMB_ACT_SIGMOID && KRAG_RERANK_IDENTITY == EMB_ACT_IDENTITY, "head activations");
int32_t krag_rerank(krag_embedder* h, int32_t n_queries, const int32_t* pair_offsets, const int32_t* tok_ids, const int32_t* tok_offsets,
                    const int32_t* seg_b, int32_t activation, int32_t top_k, int32_t* out_pos, float* out_score)
{
    return guarded([&] {
        KRAG_REQUIRE(h && pair_offsets && out_pos && out_score && n_queries >= 1, KRAG_E_INVALID, "bad argument");
        KRAG_REQUIRE(pair_offsets[n_queries] == 0 || (tok_ids && tok_offsets), KRAG_E_INVALID, "bad argument");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        embedder_rerank(h->e, n_queries, pair_offsets, tok_ids, tok_offsets, seg_b, activation, top_k, out_pos, out_score);
    });
}
int32_t krag_embedder_set_late_interaction(krag_embedder* h, int32_t dim, const float* weight, int64_t n_elems)
{
    return guarded([&] {
        KRAG_REQUIRE(h && weight, KRAG_E_INVALID, "null argument");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        embedder_set_late_interaction(h->e, dim, weight, n_elems);
    });
}
int32_t krag_late_rerank(krag_embedder* h, int32_t n_queries, int32_t query_len, const int32_t* query_tok, const int32_t* query_keys,
                         int32_t n_passages, const int32_t* passage_tok, const int32_t* passage_offsets, const uint8_t* passage_keep,
                         const int32_t* pair_offsets, const int32_t* pair_passage, int32_t top_k, int32_t* out_pos, float* out_score)
{
    return guarded([&] {
        KRAG_REQUIRE(h && query_tok && query_keys && pair_offsets && out_pos && out_score && n_queries >= 1, KRAG_E_INVALID, "bad argument");
        KRAG_REQUIRE(pair_offsets[n_queries] == 0 || (passage_tok && passage_offsets && passage_keep && pair_passage), KRAG_E_INVALID,
                     "bad argument");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        embedder_late_rerank(h->e, n_queries, query_len, query_tok, query_keys, n_passages, passage_tok, passage_offsets, passage_keep,
                             pair_offsets, pair_passage, top_k, out_pos, out_score);
    });
}
int32_t krag_debug_late_vectors(krag_embedder* h, int32_t batch, const int32_t* tok_ids, const int32_t* tok_offsets, const int32_t* key_lens,
                                float* out)
{
    return guarded([&] {
        KRAG_REQUIRE(h && tok_ids && tok_offsets && out && batch >= 1, KRAG_E_INVALID, "bad argument");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        embedder_late_vectors(h->e, batch, tok_ids, tok_offsets, key_lens, out);
    });
}
struct krag_late_store { krag_embedder* emb; LateStore* s; };
int32_t krag_embedder_set_store_budget(krag_embedder* h, int64_t bytes)
{
    return guarded([&] {
        KRAG_REQUIRE(h, KRAG_E_INVALID, "null embedder");
        embedder_set_store_budget(h->e, bytes);
    });
}
int32_t krag_late_store_create(krag_embedder* h, krag_late_store** out)
{
    return guarded([&] {
        KRAG_REQUIRE(h && out, KRAG_E_INVALID, "null argument");
        *out = new krag_late_store{h, late_store_create(h->e)};
    });
}
int32_t krag_late_store_destroy(krag_late_store* s)
{
    return guarded([&] {
        KRAG_REQUIRE(s, KRAG_E_INVALID, "null store");
        cudaSetDevice(s->emb->ctx->di.device);
        late_store_destroy(s->s);
        delete s;
    });
}
int32_t krag_late_store_append(krag_late_store* s, int32_t n, const int32_t* passage_tok, const int32_t* passage_offsets,
                               const uint8_t* passage_keep, uint8_t* stored_out)
{
    return guarded([&] {
        KRAG_REQUIRE(s && passage_tok && passage_offsets && passage_keep && stored_out && n >= 1, KRAG_E_INVALID, "bad argument");
        KRAG_CUDA(cudaSetDevice(s->emb->ctx->di.device));
        late_store_append(s->s, n, passage_tok, passage_offsets, passage_keep, stored_out);
    });
}
int32_t krag_late_store_truncate(krag_late_store* s, int64_t n_ordinals)
{
    return guarded([&] {
        KRAG_REQUIRE(s, KRAG_E_INVALID, "null store");
        KRAG_CUDA(cudaSetDevice(s->emb->ctx->di.device));
        late_store_truncate(s->s, n_ordinals);
    });
}
int32_t krag_late_store_compact(krag_late_store* s, const uint32_t* alive_bitmap, int64_t n_ordinals)
{
    return guarded([&] {
        KRAG_REQUIRE(s && (alive_bitmap || n_ordinals == 0), KRAG_E_INVALID, "bad argument");
        KRAG_CUDA(cudaSetDevice(s->emb->ctx->di.device));
        late_store_compact(s->s, alive_bitmap, n_ordinals);
    });
}
int32_t krag_late_store_stats(const krag_late_store* s, int64_t* ordinals, int64_t* stored, int64_t* rows, int64_t* device_bytes)
{
    return guarded([&] {
        KRAG_REQUIRE(s, KRAG_E_INVALID, "null store");
        int64_t v[4];
        late_store_stats(s->s, &v[0], &v[1], &v[2], &v[3]);
        if (ordinals) *ordinals = v[0];
        if (stored) *stored = v[1];
        if (rows) *rows = v[2];
        if (device_bytes) *device_bytes = v[3];
    });
}
int32_t krag_late_rerank_stored(krag_embedder* h, const krag_late_store* s, int32_t n_queries, int32_t query_len, const int32_t* query_tok,
                                const int32_t* query_keys, int32_t n_passages, const int32_t* passage_tok, const int32_t* passage_offsets,
                                const uint8_t* passage_keep, const int32_t* pair_offsets, const int32_t* pair_source, int32_t top_k,
                                int32_t* out_pos, float* out_score)
{
    return guarded([&] {
        KRAG_REQUIRE(h && s && query_tok && query_keys && pair_offsets && out_pos && out_score && n_queries >= 1, KRAG_E_INVALID, "bad argument");
        KRAG_REQUIRE(pair_offsets[n_queries] == 0 || pair_source, KRAG_E_INVALID, "bad argument");
        KRAG_REQUIRE(n_passages == 0 || (passage_tok && passage_offsets && passage_keep), KRAG_E_INVALID, "bad argument");
        KRAG_CUDA(cudaSetDevice(h->ctx->di.device));
        late_store_rerank(h->e, s->s, n_queries, query_len, query_tok, query_keys, n_passages, passage_tok, passage_offsets, passage_keep,
                          pair_offsets, pair_source, top_k, out_pos, out_score);
    });
}
int32_t krag_debug_late_store_vectors(const krag_late_store* s, int64_t ordinal, float* out, int64_t n_rows)
{
    return guarded([&] {
        KRAG_REQUIRE(s && out, KRAG_E_INVALID, "null argument");
        KRAG_CUDA(cudaSetDevice(s->emb->ctx->di.device));
        late_store_vectors(s->s, ordinal, out, n_rows);
    });
}
int32_t krag_embedder_destroy(krag_embedder* h)
{
    return guarded([&] {
        KRAG_REQUIRE(h, KRAG_E_INVALID, "null embedder");
        cudaSetDevice(h->ctx->di.device);
        embedder_destroy(h->e);
        delete h;
    });
}
static void debug_linear(krag_ctx* c, int32_t M, int32_t N, int32_t K, const float* A, const float* B, const float* bias,
                         const float* residual, int32_t gelu, const float* ln_g, const float* ln_b, float eps, float* out,
                         int32_t tile_n = 0, int32_t reps = 0, float* ms = nullptr, int planes = 2)
{
    KRAG_REQUIRE(c && A && B && bias && out && M >= 1 && N % 128 == 0 && K % 64 == 0, KRAG_E_INVALID, "bad argument (N % 128, K % 64)");
    KRAG_REQUIRE((tile_n == 0 || tile_n == 32 || tile_n == 64 || tile_n == 128 || (tile_n == 256 && planes == 1 && N % 256 == 0)) &&
                     reps >= 0 && (reps == 0 || ms),
                 KRAG_E_INVALID, "bad tile width (0, 32, 64 or 128; 256 for the fp16 GEMM with N % 256 == 0) or repeat count");
    KRAG_CUDA(cudaSetDevice(c->di.device));
    DevArray<float> dA, dB, db, dr, dC, dY, dg, dlb, ws;
    const size_t ws_floats = (size_t)4 << 20;
    dA.alloc((int64_t)M * K); dB.alloc((int64_t)N * K); db.alloc(N); dC.alloc((int64_t)M * N); ws.alloc((int64_t)ws_floats);
    KRAG_CUDA(cudaMemcpy(dA.p, A, 4 * (size_t)M * K, cudaMemcpyHostToDevice)); KRAG_CUDA(cudaMemcpy(dB.p, B, 4 * (size_t)N * K, cudaMemcpyHostToDevice));
    KRAG_CUDA(cudaMemcpy(db.p, bias, 4 * (size_t)N, cudaMemcpyHostToDevice));
    if (residual) { dr.alloc((int64_t)M * N); KRAG_CUDA(cudaMemcpy(dr.p, residual, 4 * (size_t)M * N, cudaMemcpyHostToDevice)); }
    if (ln_g) {
        dg.alloc(N); dlb.alloc(N); dY.alloc((int64_t)M * N);
        KRAG_CUDA(cudaMemcpy(dg.p, ln_g, 4 * (size_t)N, cudaMemcpyHostToDevice)); KRAG_CUDA(cudaMemcpy(dlb.p, ln_b, 4 * (size_t)N, cudaMemcpyHostToDevice));
    }
    launch_linear_f32(c->di, dA.p, dB.p, M, N, K, db.p, dr.p, gelu != 0, dC.p, dg.p, dlb.p, eps, dY.p, ws.p, ws_floats, c->admin, tile_n, reps, ms, planes);
    KRAG_CUDA(cudaStreamSynchronize(c->admin));
    KRAG_CUDA(cudaMemcpy(out, ln_g ? dY.p : dC.p, 4 * (size_t)M * N, cudaMemcpyDeviceToHost));
}

int32_t krag_debug_gemm_tf32(krag_ctx* c, int32_t M, int32_t N, int32_t K, const float* A, const float* B, const float* bias,
                             const float* residual, int32_t gelu, float* C_out, int32_t tile_n, int32_t reps, float* ms_out)
{
    return guarded([&] { debug_linear(c, M, N, K, A, B, bias, residual, gelu, nullptr, nullptr, 0.f, C_out, tile_n, reps, ms_out); });
}

int32_t krag_debug_gemm_f16(krag_ctx* c, int32_t M, int32_t N, int32_t K, const float* A, const float* B, const float* bias,
                            const float* residual, int32_t gelu, float* C_out, int32_t tile_n, int32_t reps, float* ms_out)
{
    return guarded([&] { debug_linear(c, M, N, K, A, B, bias, residual, gelu, nullptr, nullptr, 0.f, C_out, tile_n, reps, ms_out, 1); });
}

int32_t krag_debug_linear_ln(krag_ctx* c, int32_t M, int32_t N, int32_t K, const float* A, const float* B, const float* bias,
                             const float* residual, const float* ln_gamma, const float* ln_beta, float eps, float* Y_out)
{
    return guarded([&] {
        KRAG_REQUIRE(ln_gamma && ln_beta, KRAG_E_INVALID, "null LayerNorm parameters");
        debug_linear(c, M, N, K, A, B, bias, residual, 0, ln_gamma, ln_beta, eps, Y_out);
    });
}

// Own on-disk format (SURVEY.md section 5: the snapshot only needs to round-trip itself).
static const char kMagic[8] = {'K', 'R', 'A', 'G', 'I', 'D', 'X', '1'};

int32_t krag_index_persist(krag_index* ix, const char* dir)
{
    return guarded([&] {
        KRAG_REQUIRE(ix && dir, KRAG_E_INVALID, "null argument");
        std::shared_lock<std::shared_mutex> lk(ix->mu);
        require_idle(ix);
        wait_issued_searches(ix);
        KRAG_CUDA(cudaSetDevice(ix->ctx->di.device));
        mkdir(dir, 0755);
        std::string path = std::string(dir) + "/krag_index.bin";
        FILE* f = fopen((path + ".tmp").c_str(), "wb");
        KRAG_REQUIRE(f, KRAG_E_IO, "cannot open " + path + ".tmp for writing");
        auto W = [&](const void* p, size_t n) { if (n && fwrite(p, 1, n, f) != n) { fclose(f); throw ApiError{KRAG_E_IO, "short write to " + path}; } };
        int64_t hdr[8] = {ix->rows.dim, ix->rows.n, ix->nnz, ix->has_sparse ? 1 : 0, ix->committed ? ix->vocab : 0, 0, 0, 0};
        W(kMagic, 8); W(hdr, sizeof hdr);
        W(ix->node_ids.data(), sizeof(uint64_t) * (size_t)ix->rows.n);
        W(ix->alive_h.data(), sizeof(uint32_t) * (size_t)((ix->rows.n + 31) / 32));
        const int64_t chunk = 1 << 16;
        std::vector<float> rows((size_t)chunk * ix->rows.dim);
        for (int64_t r = 0; r < ix->rows.n; r += chunk) {
            int64_t m = ix->rows.n - r < chunk ? ix->rows.n - r : chunk;
            ix->rows.read(r, m, rows.data());
            W(rows.data(), sizeof(float) * (size_t)m * ix->rows.dim);
        }
        if (ix->has_sparse) {
            std::vector<int64_t> off((size_t)ix->rows.n + 1);
            std::vector<uint32_t> dl((size_t)ix->rows.n), ids((size_t)ix->nnz);
            std::vector<uint16_t> tf((size_t)ix->nnz);
            KRAG_CUDA(cudaMemcpy(off.data(), ix->toff.p, sizeof(int64_t) * off.size(), cudaMemcpyDeviceToHost));
            if (ix->rows.n) KRAG_CUDA(cudaMemcpy(dl.data(), ix->dlen.p, sizeof(uint32_t) * dl.size(), cudaMemcpyDeviceToHost));
            if (ix->nnz) {
                KRAG_CUDA(cudaMemcpy(ids.data(), ix->tid.p, sizeof(uint32_t) * ids.size(), cudaMemcpyDeviceToHost));
                KRAG_CUDA(cudaMemcpy(tf.data(), ix->ttf.p, sizeof(uint16_t) * tf.size(), cudaMemcpyDeviceToHost));
            }
            W(off.data(), sizeof(int64_t) * off.size()); W(dl.data(), sizeof(uint32_t) * dl.size());
            W(ids.data(), sizeof(uint32_t) * ids.size()); W(tf.data(), sizeof(uint16_t) * tf.size());
        }
        KRAG_REQUIRE(fclose(f) == 0, KRAG_E_IO, "close failed for " + path);
        KRAG_REQUIRE(rename((path + ".tmp").c_str(), path.c_str()) == 0, KRAG_E_IO, "rename failed for " + path);
    });
}

int32_t krag_index_load(krag_ctx* c, const char* name, const char* dir, krag_index** out)
{
    krag_index* ix = nullptr;
    int32_t rc = guarded([&] {
        KRAG_REQUIRE(c && name && dir && out, KRAG_E_INVALID, "null argument");
        std::string path = std::string(dir) + "/krag_index.bin";
        FILE* f = fopen(path.c_str(), "rb");
        KRAG_REQUIRE(f, KRAG_E_IO, "cannot open " + path);
        auto R = [&](void* p, size_t n) { if (n && fread(p, 1, n, f) != n) { fclose(f); throw ApiError{KRAG_E_IO, "short read from " + path}; } };
        char magic[8]; int64_t hdr[8];
        R(magic, 8); R(hdr, sizeof hdr);
        if (memcmp(magic, kMagic, 8) != 0) { fclose(f); throw ApiError{KRAG_E_IO, path + " is not a krag index snapshot"}; }
        const int64_t dim = hdr[0], n = hdr[1], nnz = hdr[2], sparse = hdr[3], vocab = hdr[4];
        int32_t rc2 = krag_index_create(c, name, (int32_t)dim, &ix);
        if (rc2 != KRAG_OK) { fclose(f); throw ApiError{rc2, g_err}; }
        std::vector<uint64_t> ids((size_t)n);
        std::vector<uint32_t> alive((size_t)((n + 31) / 32));
        R(ids.data(), sizeof(uint64_t) * ids.size()); R(alive.data(), sizeof(uint32_t) * alive.size());
        std::vector<float> rows((size_t)n * dim);
        R(rows.data(), sizeof(float) * rows.size());
        std::vector<int64_t> off; std::vector<uint32_t> dl, tids; std::vector<uint16_t> tf;
        if (sparse) {
            off.resize((size_t)n + 1); dl.resize((size_t)n); tids.resize((size_t)nnz); tf.resize((size_t)nnz);
            R(off.data(), sizeof(int64_t) * off.size()); R(dl.data(), sizeof(uint32_t) * dl.size());
            R(tids.data(), sizeof(uint32_t) * tids.size()); R(tf.data(), sizeof(uint16_t) * tf.size());
        }
        fclose(f);
        if (n > 0) {
            rc2 = krag_index_add(ix, n, ids.data(), rows.data(), sparse ? off.data() : nullptr, sparse ? tids.data() : nullptr,
                                 sparse ? tf.data() : nullptr, sparse ? dl.data() : nullptr);
            if (rc2 != KRAG_OK) throw ApiError{rc2, g_err};
            std::vector<uint64_t> dead;
            for (int64_t r = 0; r < n; ++r) if (!((alive[(size_t)(r >> 5)] >> (r & 31)) & 1u)) dead.push_back(ids[(size_t)r]);
            if (!dead.empty()) { rc2 = krag_index_remove(ix, (int64_t)dead.size(), dead.data(), nullptr); if (rc2 != KRAG_OK) throw ApiError{rc2, g_err}; }
        }
        if (sparse && vocab > 0) { rc2 = krag_index_commit(ix, vocab); if (rc2 != KRAG_OK) throw ApiError{rc2, g_err}; }
        *out = ix;
    });
    if (rc != KRAG_OK && ix) { std::string keep = g_err; krag_index_drop(ix); set_error(keep); }
    return rc;
}

}  // extern "C"
