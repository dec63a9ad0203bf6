// postings_merge.cu -- incremental BM25 commit and compaction: the committed postings are merged with the rows added since,
// or remapped to compacted row numbers, instead of being rebuilt from every raw term list.
//
// A base list never gains a row (rows added since the base have higher row numbers and go behind it) and only loses rows that
// died (rows never come back to life), so a term's new list is its base list filtered by the alive bitmap, in base order,
// followed by the term's live new rows.  Each pass below reads the base postings once, in fixed blocks of PM_BLOCK postings;
// a block finds the terms of its postings from the offsets (one binary search per thread inside the block's term bracket,
// then a forward walk), so no per-posting term array is needed.  A block may straddle term boundaries and one term may span
// thousands of blocks.
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include "engine.h"

namespace krag {

namespace {

constexpr int PM_THREADS = 256;
constexpr int PM_ITEMS = 8;                                   // consecutive postings per thread
constexpr int64_t PM_BLOCK = (int64_t)PM_THREADS * PM_ITEMS;  // postings per block

int64_t pm_blocks(int64_t nnz) { return (nnz + PM_BLOCK - 1) / PM_BLOCK; }

// largest t in [lo, hi] with off[t] <= p: the term whose list holds posting p (empty terms before it share its offset)
__device__ __forceinline__ int64_t term_of(const int64_t* __restrict__ off, int64_t lo, int64_t hi, int64_t p)
{
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (off[mid] <= p) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// terms of the first and the last posting of this block -> s_t[0], s_t[1] (every thread of the block calls it)
__device__ __forceinline__ void block_terms(const int64_t* __restrict__ off, int64_t vocab, int64_t nnz, int64_t p0, int64_t* s_t)
{
    if (threadIdx.x == 0) {
        const int64_t last = (p0 + PM_BLOCK < nnz ? p0 + PM_BLOCK : nnz) - 1;
        s_t[0] = term_of(off, 0, vocab - 1, p0);
        s_t[1] = term_of(off, s_t[0], vocab - 1, last);
    }
    __syncthreads();
}

// live base postings per term (per_term += ...) and per block (block_cnt); a block inside one term adds once
__global__ void __launch_bounds__(PM_THREADS)
survivor_count_kernel(const int64_t* __restrict__ off, const uint32_t* __restrict__ doc, const uint32_t* __restrict__ alive,
                      int64_t nnz, int64_t vocab, uint32_t* __restrict__ per_term, int64_t* __restrict__ block_cnt)
{
    __shared__ int64_t s_t[2];
    __shared__ uint32_t s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    const int64_t p0 = (int64_t)blockIdx.x * PM_BLOCK;
    block_terms(off, vocab, nnz, p0, s_t);
    const bool one_term = s_t[0] == s_t[1];
    const int64_t first = p0 + (int64_t)threadIdx.x * PM_ITEMS;
    uint32_t total = 0;
    if (first < nnz) {
        int64_t t = one_term ? s_t[0] : term_of(off, s_t[0], s_t[1], first);
        uint32_t run = 0;
#pragma unroll
        for (int k = 0; k < PM_ITEMS; ++k) {
            const int64_t p = first + k;
            if (p >= nnz) break;
            if (!one_term) {
                while (off[t + 1] <= p) {
                    if (run) { atomicAdd(&per_term[t], run); run = 0; }
                    ++t;
                }
            }
            const uint32_t ok = (alive == nullptr || bit_test(alive, doc[p])) ? 1u : 0u;
            run += ok;
            total += ok;
        }
        if (!one_term && run) atomicAdd(&per_term[t], run);
    }
    total = __reduce_add_sync(0xffffffffu, total);
    if ((threadIdx.x & 31) == 0 && total) atomicAdd(&s_cnt, total);
    __syncthreads();
    if (threadIdx.x == 0) {
        block_cnt[blockIdx.x] = s_cnt;
        if (one_term && s_cnt) atomicAdd(&per_term[s_t[0]], s_cnt);
    }
}

// survivor k of term t (base order) -> out_off[t] + k.  k = (live base postings before it) - (live base postings before t).
// REMAP: doc -> rank[doc], tf and score copied; otherwise rescored with the full build's arithmetic.
template <bool REMAP>
__global__ void __launch_bounds__(PM_THREADS)
survivor_write_kernel(const int64_t* __restrict__ off, const uint32_t* __restrict__ doc, const uint16_t* __restrict__ tf,
                      const float* __restrict__ score, int64_t nnz, int64_t vocab, const uint32_t* __restrict__ alive,
                      const int64_t* __restrict__ block_off, const int64_t* __restrict__ before, const int64_t* __restrict__ out_off,
                      const uint32_t* __restrict__ rank, const uint32_t* __restrict__ doc_len, const float* __restrict__ idf,
                      double avgdl, uint32_t* __restrict__ out_doc, uint16_t* __restrict__ out_tf, float* __restrict__ out_score)
{
    typedef cub::BlockScan<uint32_t, PM_THREADS> Scan;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int64_t s_t[2];
    const int64_t p0 = (int64_t)blockIdx.x * PM_BLOCK;
    block_terms(off, vocab, nnz, p0, s_t);
    const int64_t first = p0 + (int64_t)threadIdx.x * PM_ITEMS;
    bool ok[PM_ITEMS];
    uint32_t c = 0;
#pragma unroll
    for (int k = 0; k < PM_ITEMS; ++k) {
        ok[k] = first + k < nnz && (alive == nullptr || bit_test(alive, doc[first + k]));
        c += ok[k] ? 1u : 0u;
    }
    uint32_t excl;
    Scan(tmp).ExclusiveSum(c, excl);
    if (c == 0) return;
    int64_t s = block_off[blockIdx.x] + excl;                 // live base postings before this thread's first item
    int64_t t = term_of(off, s_t[0], s_t[1], first);
#pragma unroll
    for (int k = 0; k < PM_ITEMS; ++k) {
        const int64_t p = first + k;
        if (p >= nnz) break;
        while (off[t + 1] <= p) ++t;
        if (!ok[k]) continue;
        const int64_t at = out_off[t] + (s - before[t]);
        const uint32_t d = doc[p];
        if (REMAP) {
            out_doc[at] = rank[d];
            out_tf[at] = tf[p];
            out_score[at] = score[p];
        } else {
            const uint16_t f = tf[p];
            out_doc[at] = d;
            out_tf[at] = f;
            out_score[at] = bm25_posting_score(idf[t], f, doc_len[d], avgdl);
        }
        ++s;
    }
}

__global__ void delta_write_kernel(const uint32_t* __restrict__ keys, const uint64_t* __restrict__ vals, int64_t q_base, int64_t m,
                                   const int64_t* __restrict__ delta_off, const uint32_t* __restrict__ survivors,
                                   const int64_t* __restrict__ out_off, const uint32_t* __restrict__ doc_len,
                                   const float* __restrict__ idf, double avgdl, uint32_t* __restrict__ out_doc,
                                   uint16_t* __restrict__ out_tf, float* __restrict__ out_score)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t t = keys[i];
        const uint64_t v = vals[i];
        const uint32_t d = (uint32_t)(v >> 16), f = (uint32_t)(v & 0xffffu);
        const int64_t at = out_off[t] + survivors[t] + (q_base + i - delta_off[t]);
        out_doc[at] = d;
        out_tf[at] = (uint16_t)f;
        out_score[at] = bm25_posting_score(idf[t], f, doc_len[d], avgdl);
    }
}

// the boundary rows of the frequent terms, as tile_index_kernel writes them during a full build
__global__ void __launch_bounds__(PM_THREADS)
tile_fill_kernel(const int64_t* __restrict__ off, const uint32_t* __restrict__ doc, int64_t nnz, int64_t vocab,
                 const int32_t* __restrict__ slot, int64_t n_tiles, uint32_t* __restrict__ tile_off)
{
    __shared__ int64_t s_t[2];
    const int64_t p0 = (int64_t)blockIdx.x * PM_BLOCK;
    block_terms(off, vocab, nnz, p0, s_t);
    const int64_t first = p0 + (int64_t)threadIdx.x * PM_ITEMS;
    if (first >= nnz) return;
    int64_t t = term_of(off, s_t[0], s_t[1], first);
    for (int k = 0; k < PM_ITEMS; ++k) {
        const int64_t p = first + k;
        if (p >= nnz) break;
        while (off[t + 1] <= p) ++t;
        const int32_t sl = slot[t];
        if (sl < 0) continue;
        const int64_t b = off[t], e = off[t + 1];
        const int64_t i = p - b;
        const int64_t tile_d = doc[p] / BM25_SUB_DOCS;
        const int64_t prev = (i == 0) ? -1 : (int64_t)(doc[p - 1] / BM25_SUB_DOCS);
        uint32_t* row = tile_off + (int64_t)sl * (n_tiles + 1);
        for (int64_t tl = prev + 1; tl <= tile_d; ++tl) row[tl] = (uint32_t)i;
        if (p == e - 1) for (int64_t tl = tile_d + 1; tl <= n_tiles; ++tl) row[tl] = (uint32_t)(e - b);
    }
}

__global__ void live_stats_kernel(const uint32_t* __restrict__ doc_len, const uint32_t* __restrict__ alive, int64_t n_rows,
                                  unsigned long long* __restrict__ out /*[2]: rows, length*/)
{
    unsigned long long rows = 0, len = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x)
        if (alive == nullptr || bit_test(alive, (uint32_t)r)) { ++rows; len += doc_len[r]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        rows += __shfl_xor_sync(0xffffffffu, rows, o);
        len += __shfl_xor_sync(0xffffffffu, len, o);
    }
    if ((threadIdx.x & 31) == 0 && rows) { atomicAdd(&out[0], rows); atomicAdd(&out[1], len); }
}

__global__ void add_u32_kernel(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, int64_t n, uint32_t* __restrict__ out)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = a[i] + b[i];
}

__global__ void rank_of_rows_kernel(const uint32_t* __restrict__ src, int64_t n_live, uint32_t* __restrict__ rank)
{
    for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < n_live; d += (int64_t)gridDim.x * blockDim.x)
        rank[src[d]] = (uint32_t)d;
}

unsigned grid_of(int64_t threads)
{
    const int64_t b = (threads + 255) / 256;
    return (unsigned)(b < 1 ? 1 : (b > 132 * 16 ? 132 * 16 : b));
}

}  // namespace

void count_survivors(const Postings& base, const uint32_t* alive, int64_t vocab, SurvivorCounts& sc, cudaStream_t st)
{
    const int64_t nb = pm_blocks(base.nnz);
    if (nb >= ((int64_t)1 << 31)) throw std::runtime_error("postings merge: too many postings on one shard");
    sc.per_term.alloc(vocab);
    sc.block_off.alloc(nb > 0 ? nb : 1);
    DevArray<int64_t> block_cnt;
    block_cnt.alloc(nb > 0 ? nb : 1);
    KRAG_CUDA(cudaMemsetAsync(sc.per_term.p, 0, sizeof(uint32_t) * (size_t)vocab, st));
    if (nb > 0) {
        survivor_count_kernel<<<(unsigned)nb, PM_THREADS, 0, st>>>(base.off.p, base.doc.p, alive, base.nnz, base.vocab,
                                                                  sc.per_term.p, block_cnt.p);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        size_t bytes = 0;
        KRAG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, block_cnt.p, sc.block_off.p, (int)nb, st));
        DevArray<unsigned char> tmp;
        tmp.alloc(bytes ? (int64_t)bytes : 1);
        KRAG_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, block_cnt.p, sc.block_off.p, (int)nb, st));
        count_launch();
    }
    df_offsets(sc.per_term.p, vocab, sc.before, nullptr, st);
}

void write_survivors(const Postings& base, const uint32_t* alive, const SurvivorCounts& sc, const int64_t* out_off,
                     const uint32_t* rank, const uint32_t* doc_len, const float* idf, double avgdl, Postings& out, cudaStream_t st)
{
    const int64_t nb = pm_blocks(base.nnz);
    if (nb == 0) return;
    if (rank)
        survivor_write_kernel<true><<<(unsigned)nb, PM_THREADS, 0, st>>>(base.off.p, base.doc.p, base.tf.p, base.score.p, base.nnz,
            base.vocab, alive, sc.block_off.p, sc.before.p, out_off, rank, doc_len, idf, avgdl, out.doc.p, out.tf.p, out.score.p);
    else
        survivor_write_kernel<false><<<(unsigned)nb, PM_THREADS, 0, st>>>(base.off.p, base.doc.p, base.tf.p, base.score.p, base.nnz,
            base.vocab, alive, sc.block_off.p, sc.before.p, out_off, rank, doc_len, idf, avgdl, out.doc.p, out.tf.p, out.score.p);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

void write_delta(const uint32_t* keys, const uint64_t* vals, int64_t q_base, int64_t m, const int64_t* delta_off,
                 const SurvivorCounts& sc, const int64_t* out_off, const uint32_t* doc_len, const float* idf, double avgdl,
                 Postings& out, cudaStream_t st)
{
    if (m == 0) return;
    delta_write_kernel<<<grid_of(m), 256, 0, st>>>(keys, vals, q_base, m, delta_off, sc.per_term.p, out_off, doc_len, idf, avgdl,
                                                   out.doc.p, out.tf.p, out.score.p);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

void fill_tile_index(Postings& out, cudaStream_t st)
{
    const int64_t nb = pm_blocks(out.nnz);
    if (nb == 0 || out.n_slots == 0) return;
    tile_fill_kernel<<<(unsigned)nb, PM_THREADS, 0, st>>>(out.off.p, out.doc.p, out.nnz, out.vocab, out.tile_slot.p, out.n_tiles,
                                                          out.tile_off.p);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

void live_doc_stats(const uint32_t* doc_len, const uint32_t* alive, int64_t n_rows, int64_t* n_live, int64_t* total_len,
                    cudaStream_t st)
{
    *n_live = 0;
    *total_len = 0;
    if (n_rows == 0) return;
    DevArray<unsigned long long> acc;
    acc.alloc(2);
    KRAG_CUDA(cudaMemsetAsync(acc.p, 0, 2 * sizeof(unsigned long long), st));
    live_stats_kernel<<<grid_of(n_rows), 256, 0, st>>>(doc_len, alive, n_rows, acc.p);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    unsigned long long h[2];
    KRAG_CUDA(cudaMemcpyAsync(h, acc.p, sizeof h, cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    *n_live = (int64_t)h[0];
    *total_len = (int64_t)h[1];
}

void launch_add_u32(const uint32_t* a, const uint32_t* b, int64_t n, uint32_t* out, cudaStream_t st)
{
    if (n == 0) return;
    add_u32_kernel<<<grid_of(n), 256, 0, st>>>(a, b, n, out);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

void launch_rank_of_rows(const uint32_t* src, int64_t n_live, uint32_t* rank, cudaStream_t st)
{
    if (n_live == 0) return;
    rank_of_rows_kernel<<<grid_of(n_live), 256, 0, st>>>(src, n_live, rank);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

}  // namespace krag
