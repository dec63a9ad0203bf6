// compact.cu -- krag_index_compact: tombstoned rows removed in place.  Live row r moves down to rank(r) <= r (its number
// of live predecessors), so live rows keep their order and every tie-break by ordinal is unchanged.
//
// The moves run in windows of destination rows, in ascending order, on one stream.  A window whose destination range ends at
// or below its first source row reads nothing it writes and is gathered directly; any other window is gathered into a bounded
// staging buffer and copied down from there.  Either way, a window only overwrites source rows of earlier windows (already
// moved) or dead rows, since every later window reads at or above its own first source row, which is >= its destination.
#include <cub/cub.cuh>

#include <algorithm>

#include "engine.h"

namespace krag {

namespace {

// the alive bits of word w (bits past n_rows cleared)
__device__ __forceinline__ uint32_t live_word(const uint32_t* __restrict__ alive, int64_t w, int64_t n_rows)
{
    uint32_t v = alive[w];
    const int64_t tail = n_rows - w * 32;
    if (tail < 32) v &= (1u << tail) - 1u;
    return v;
}

__global__ void word_popc_kernel(const uint32_t* __restrict__ alive, int64_t words, int64_t n_rows, int64_t* __restrict__ cnt)
{
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w <= words; w += (int64_t)gridDim.x * blockDim.x)
        cnt[w] = w < words ? __popc(live_word(alive, w, n_rows)) : 0;
}

// src[rank(r)] = r for every live row r; rank = live rows in earlier words + live rows below r in its word
__global__ void src_rows_kernel(const uint32_t* __restrict__ alive, const int64_t* __restrict__ word_rank, int64_t n_rows,
                                uint32_t* __restrict__ src)
{
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t w = live_word(alive, r >> 5, n_rows);
        const uint32_t bit = (uint32_t)(r & 31);
        if ((w >> bit) & 1u) src[word_rank[r >> 5] + __popc(w & ((1u << bit) - 1u))] = (uint32_t)r;
    }
}

// term-list length of each destination row (and a trailing 0, so the exclusive scan ends with the new nnz)
__global__ void new_len_kernel(const int64_t* __restrict__ toff, const uint32_t* __restrict__ src, int64_t n_live,
                               int64_t* __restrict__ len)
{
    for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d <= n_live; d += (int64_t)gridDim.x * blockDim.x) {
        if (d == n_live) { len[d] = 0; continue; }
        const uint32_t s = src[d];
        len[d] = toff[s + 1] - toff[s];
    }
}

// dst row i <- src row src_row[d0 + i], i in [0, n); rows of row_vecs V-sized words.  One thread per row for single-word rows,
// one warp per row otherwise (16-byte accesses, coalesced across the warp).
template <class V>
__global__ void __launch_bounds__(256)
gather_rows_kernel(const V* __restrict__ src, V* __restrict__ dst, const uint32_t* __restrict__ src_row, int64_t d0, int64_t n,
                   int64_t row_vecs)
{
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (int64_t)gridDim.x * blockDim.x;
    if (row_vecs == 1) {
        for (int64_t i = tid; i < n; i += nthreads) dst[i] = src[src_row[d0 + i]];
        return;
    }
    const int lane = threadIdx.x & 31;
    for (int64_t i = tid >> 5; i < n; i += nthreads >> 5) {
        const V* s = src + (int64_t)src_row[d0 + i] * row_vecs;
        V* o = dst + i * row_vecs;
        for (int64_t j = lane; j < row_vecs; j += 32) o[j] = s[j];
    }
}

// term lists of destination rows [d0, d0 + n): one warp per row; entries land at toff_new[d] - e0 of the destination arrays
__global__ void __launch_bounds__(256)
gather_terms_kernel(const uint32_t* __restrict__ tid, const uint16_t* __restrict__ ttf, const int64_t* __restrict__ toff_old,
                    const int64_t* __restrict__ toff_new, const uint32_t* __restrict__ src_row, int64_t d0, int64_t n, int64_t e0,
                    uint32_t* __restrict__ tid_dst, uint16_t* __restrict__ ttf_dst)
{
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
        const uint32_t s = src_row[d0 + i];
        const int64_t b = toff_old[s], len = toff_old[s + 1] - b, o = toff_new[d0 + i] - e0;
        for (int64_t j = lane; j < len; j += 32) { tid_dst[o + j] = tid[b + j]; ttf_dst[o + j] = ttf[b + j]; }
    }
}

__global__ void max_bits_kernel(const float* __restrict__ x, int64_t n, uint32_t* __restrict__ max_bits)
{
    uint32_t m = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        m = max(m, __float_as_uint(x[i]));   // x >= 0: the bit patterns order as the values
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(max_bits, m);
}

unsigned grid_for(int64_t threads)
{
    const int64_t b = (threads + 255) / 256;
    return (unsigned)(b < 1 ? 1 : (b > 132 * 16 ? 132 * 16 : b));
}

template <class T>
void exclusive_sum(const T* in, T* out, int64_t n, cudaStream_t st)
{
    size_t bytes = 0;
    KRAG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, st));
    DevArray<unsigned char> tmp;
    tmp.alloc(bytes ? (int64_t)bytes : 1);
    KRAG_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, in, out, n, st));
    count_launch();
}

}  // namespace

void compact_plan(const uint32_t* alive, int64_t n_rows, const int64_t* toff, CompactPlan& plan, cudaStream_t st)
{
    const int64_t words = (n_rows + 31) / 32;
    plan.n_rows = n_rows;
    {
        DevArray<int64_t> cnt, rank;
        cnt.alloc(words + 1);
        rank.alloc(words + 1);
        word_popc_kernel<<<grid_for(words + 1), 256, 0, st>>>(alive, words, n_rows, cnt.p);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        exclusive_sum(cnt.p, rank.p, words + 1, st);
        KRAG_CUDA(cudaMemcpyAsync(&plan.n_live, rank.p + words, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
        plan.src.alloc(plan.n_live > 0 ? plan.n_live : 1);
        src_rows_kernel<<<grid_for(n_rows), 256, 0, st>>>(alive, rank.p, n_rows, plan.src.p);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        plan.h_src.resize((size_t)plan.n_live);
        if (plan.n_live > 0)
            KRAG_CUDA(cudaMemcpyAsync(plan.h_src.data(), plan.src.p, sizeof(uint32_t) * (size_t)plan.n_live, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
    }
    plan.first = 0;
    while (plan.first < plan.n_live && plan.h_src[(size_t)plan.first] == (uint32_t)plan.first) ++plan.first;
    int64_t stage_bytes = COMPACT_STAGE_BYTES;
    if (toff) {
        DevArray<int64_t> len;
        len.alloc(plan.n_live + 1);
        plan.toff_new.alloc(plan.n_live + 1);
        new_len_kernel<<<grid_for(plan.n_live + 1), 256, 0, st>>>(toff, plan.src.p, plan.n_live, len.p);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        exclusive_sum(len.p, plan.toff_new.p, plan.n_live + 1, st);
        plan.h_toff_old.resize((size_t)n_rows + 1);
        plan.h_toff_new.resize((size_t)plan.n_live + 1);
        KRAG_CUDA(cudaMemcpyAsync(plan.h_toff_old.data(), toff, sizeof(int64_t) * (size_t)(n_rows + 1), cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaMemcpyAsync(plan.h_toff_new.data(), plan.toff_new.p, sizeof(int64_t) * (size_t)(plan.n_live + 1),
                                  cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
        // a term list longer than the staging buffer is one window of its own: the buffer holds at least one
        int64_t longest = 0;
        for (int64_t d = plan.first; d < plan.n_live; ++d)
            longest = std::max(longest, plan.h_toff_new[(size_t)d + 1] - plan.h_toff_new[(size_t)d]);
        stage_bytes = std::max(stage_bytes, longest * COMPACT_TERM_BYTES);
    }
    plan.stage.alloc(stage_bytes);
}

int64_t compact_rows(void* base, int64_t row_bytes, const CompactPlan& plan, cudaStream_t st)
{
    if (plan.first >= plan.n_live) return 0;
    const bool v16 = row_bytes % 16 == 0;
    const int64_t row_vecs = v16 ? row_bytes / 16 : row_bytes / 4;
    const int64_t W = std::max<int64_t>(1, plan.stage.cap / row_bytes);
    char* b = static_cast<char*>(base);
    for (int64_t d0 = plan.first; d0 < plan.n_live; d0 += W) {
        const int64_t d1 = std::min(plan.n_live, d0 + W), n = d1 - d0;
        const bool direct = d1 <= (int64_t)plan.h_src[(size_t)d0];
        void* dst = direct ? (void*)(b + d0 * row_bytes) : (void*)plan.stage.p;
        const unsigned grid = grid_for(row_vecs == 1 ? n : n * 32);
        if (v16)
            gather_rows_kernel<uint4><<<grid, 256, 0, st>>>((const uint4*)b, (uint4*)dst, plan.src.p, d0, n, row_vecs);
        else
            gather_rows_kernel<uint32_t><<<grid, 256, 0, st>>>((const uint32_t*)b, (uint32_t*)dst, plan.src.p, d0, n, row_vecs);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        if (!direct)
            KRAG_CUDA(cudaMemcpyAsync(b + d0 * row_bytes, plan.stage.p, (size_t)(n * row_bytes), cudaMemcpyDeviceToDevice, st));
    }
    return (plan.n_live - plan.first) * row_bytes;
}

int64_t compact_terms(uint32_t* tid, uint16_t* ttf, const int64_t* toff_old, const CompactPlan& plan, cudaStream_t st)
{
    if (plan.first >= plan.n_live) return 0;
    const std::vector<int64_t>& to = plan.h_toff_old;
    const std::vector<int64_t>& tn = plan.h_toff_new;
    const int64_t cap = plan.stage.cap / COMPACT_TERM_BYTES;
    uint32_t* s_tid = reinterpret_cast<uint32_t*>(plan.stage.p);
    uint16_t* s_ttf = reinterpret_cast<uint16_t*>(plan.stage.p + cap * sizeof(uint32_t));
    for (int64_t d0 = plan.first; d0 < plan.n_live;) {
        // the longest run of rows from d0 whose entries fit the staging buffer (at least one row)
        int64_t d1 = (int64_t)(std::upper_bound(tn.begin() + d0 + 1, tn.end(), tn[(size_t)d0] + cap) - tn.begin()) - 1;
        d1 = std::min(plan.n_live, std::max(d1, d0 + 1));
        const int64_t e0 = tn[(size_t)d0], ne = tn[(size_t)d1] - e0;
        const bool direct = tn[(size_t)d1] <= to[plan.h_src[(size_t)d0]];
        if (ne > 0) {
            gather_terms_kernel<<<grid_for((d1 - d0) * 32), 256, 0, st>>>(tid, ttf, toff_old, plan.toff_new.p, plan.src.p, d0, d1 - d0,
                                                                           direct ? 0 : e0, direct ? tid : s_tid, direct ? ttf : s_ttf);
            KRAG_CUDA(cudaGetLastError());
            count_launch();
            if (!direct) {
                KRAG_CUDA(cudaMemcpyAsync(tid + e0, s_tid, sizeof(uint32_t) * (size_t)ne, cudaMemcpyDeviceToDevice, st));
                KRAG_CUDA(cudaMemcpyAsync(ttf + e0, s_ttf, sizeof(uint16_t) * (size_t)ne, cudaMemcpyDeviceToDevice, st));
            }
        }
        d0 = d1;
    }
    return (tn[(size_t)plan.n_live] - tn[(size_t)plan.first]) * COMPACT_TERM_BYTES;
}

void launch_max_bits(const float* x, int64_t n, uint32_t* max_bits, cudaStream_t st)
{
    KRAG_CUDA(cudaMemsetAsync(max_bits, 0, sizeof(uint32_t), st));
    if (n == 0) return;
    max_bits_kernel<<<grid_for(n), 256, 0, st>>>(x, n, max_bits);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

}  // namespace krag
