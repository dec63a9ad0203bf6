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

// ---- redeal kernels
constexpr uint32_t REDEAL_STAY = 0xFFFFFFFFu;   // sort key of rows that do not move (dead, or below the first dead ordinal)

// *first = lowest ordinal m * G + t of a zero bit over all shards' words (dead row, or padding: ordinal >= the row count)
__global__ void first_dead_kernel(const uint32_t* __restrict__ alive, int G, int64_t words, unsigned long long* first)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < G * words; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t z = ~alive[i];
        if (!z) continue;
        const int64_t t = i / words, m = (i % words) * 32 + (__ffs(z) - 1);
        atomicMin(first, (unsigned long long)(m * G + t));
    }
}

// live rows among shard t's first m rows; wscan = exclusive scan of the per-word popcounts of all shards' words
__device__ __forceinline__ int64_t live_below(const uint32_t* __restrict__ alive, const int64_t* __restrict__ wscan, int64_t words,
                                              int64_t t, int64_t m)
{
    const int64_t w = m >> 5;
    int64_t c = wscan[t * words + w] - wscan[t * words];
    if (m & 31) c += __popc(alive[t * words + w] & ((1u << (m & 31)) - 1u));
    return c;
}

// every live row (t, m) of every shard: its new ordinal, window and destination.  This shard's rows get their sort key and
// rank and fill the send tables; rows bound for this shard fill the receive table.
__global__ void redeal_rank_kernel(const uint32_t* __restrict__ alive, const int64_t* __restrict__ wscan, int G, int s, int64_t words,
                                   int64_t first, int64_t window_rows, const int64_t* __restrict__ toff, uint32_t* __restrict__ key,
                                   uint32_t* __restrict__ rank_out, uint32_t* __restrict__ iota, int64_t n_rows,
                                   unsigned long long* send_rows, unsigned long long* send_ents, unsigned long long* recv_rows)
{
    const int64_t bits = (int64_t)G * words * 32;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < bits; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = i / (words * 32), m = i % (words * 32);
        if (t == s && m < n_rows) { key[m] = REDEAL_STAY; iota[m] = (uint32_t)m; }
        if (!((alive[t * words + (m >> 5)] >> (m & 31)) & 1u)) continue;
        int64_t rank = 0;
        for (int u = 0; u < G; ++u) rank += live_below(alive, wscan, words, u, u < t ? m + 1 : m);
        if (t == s) rank_out[m] = (uint32_t)rank;
        if (rank < first) continue;
        const int64_t k = (rank - first) / window_rows, d = rank % G;
        if (t == s) {
            key[m] = (uint32_t)(k * G + d);
            atomicAdd(send_rows + k * G + d, 1ull);
            if (toff) atomicAdd(send_ents + k * G + d, (unsigned long long)(toff[m + 1] - toff[m]));
        }
        if (d == s) atomicAdd(recv_rows + k * G + t, 1ull);
    }
}

// one warp per row of the window's send segment: payload header, scalars and rows; the term entries into ents
__global__ void __launch_bounds__(256)
redeal_pack_kernel(RedealRows v, const uint32_t* __restrict__ send_row, const uint32_t* __restrict__ send_key,
                   const uint32_t* __restrict__ rank, const int64_t* __restrict__ send_ent, const int64_t* __restrict__ seg_ent, int G,
                   int64_t p0, int64_t n, int64_t row_vecs, uint4* __restrict__ out, uint2* __restrict__ ents)
{
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t e0 = send_ent[p0];
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
        const int64_t p = p0 + i;
        const uint32_t r = send_row[p];
        const int64_t b = v.toff ? v.toff[r] : 0, len = v.toff ? v.toff[r + 1] - b : 0;
        uint4* o = out + i * row_vecs;
        if (lane == 0) {
            const int64_t in_chunk = send_ent[p] - seg_ent[send_key[p]];
            o[0] = make_uint4(rank[r] / (uint32_t)G, (uint32_t)len, (uint32_t)in_chunk, (uint32_t)((uint64_t)in_chunk >> 32));
            o[1] = make_uint4(v.dlen ? v.dlen[r] : 0u, __float_as_uint(v.xnorm[r]), v.xres ? __float_as_uint(v.xres[r]) : 0u, 0u);
        }
        const int64_t xv = v.dpad / 4, hv = v.dpad / 8;
        const uint4* xs = reinterpret_cast<const uint4*>(v.x + (int64_t)r * v.dpad);
        for (int64_t j = lane; j < xv; j += 32) o[2 + j] = xs[j];
        if (v.xh) {
            const uint4* hs = reinterpret_cast<const uint4*>(v.xh + (int64_t)r * v.dpad);
            for (int64_t j = lane; j < hv; j += 32) o[2 + xv + j] = hs[j];
        }
        uint2* e = ents + (send_ent[p] - e0);
        for (int64_t j = lane; j < len; j += 32) e[j] = make_uint2(v.tid[b + j], (uint32_t)v.ttf[b + j]);
    }
}

// one warp per received row: scalars and rows to the destination row, its term count to lens[row - j0]
__global__ void __launch_bounds__(256)
redeal_unpack_rows_kernel(RedealRows v, const uint4* __restrict__ in, int64_t n, int64_t row_vecs, int64_t j0, int64_t* __restrict__ lens)
{
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
        const uint4* h = in + i * row_vecs;
        const uint4 hd = h[0];
        const int64_t j = hd.x;
        if (lane == 0) {
            const uint4 sc = h[1];
            lens[j - j0] = hd.y;
            if (v.dlen) v.dlen[j] = sc.x;
            v.xnorm[j] = __uint_as_float(sc.y);
            if (v.xres) v.xres[j] = __uint_as_float(sc.z);
        }
        const int64_t xv = v.dpad / 4, hv = v.dpad / 8;
        uint4* xd = reinterpret_cast<uint4*>(v.x + j * v.dpad);
        for (int64_t c = lane; c < xv; c += 32) xd[c] = h[2 + c];
        if (v.xh) {
            uint4* hdst = reinterpret_cast<uint4*>(v.xh + j * v.dpad);
            for (int64_t c = lane; c < hv; c += 32) hdst[c] = h[2 + xv + c];
        }
    }
}

// one warp per received row: its entries (sender t's chunk starts at ent_disp[t]) to the new term arrays at toff_new[row]
__global__ void __launch_bounds__(256)
redeal_unpack_terms_kernel(const uint4* __restrict__ in, int64_t n, int64_t row_vecs, const uint2* __restrict__ ents,
                           const int64_t* __restrict__ row_disp, const int64_t* __restrict__ ent_disp, int G,
                           const int64_t* __restrict__ toff_new, uint32_t* __restrict__ tid, uint16_t* __restrict__ ttf)
{
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
        const uint4 hd = in[i * row_vecs];
        const int64_t len = hd.y;
        if (len == 0) continue;
        int t = 0;
        while (t + 1 < G && row_disp[t + 1] <= i) ++t;       // the sender: received rows are grouped by sender
        const uint2* e = ents + ent_disp[t] + (int64_t)(((uint64_t)hd.w << 32) | hd.z);
        const int64_t o = toff_new[hd.x];
        for (int64_t j = lane; j < len; j += 32) {
            const uint2 x = e[j];
            tid[o + j] = x.x;
            ttf[o + j] = (uint16_t)x.y;
        }
    }
}

int64_t ceil_rows(int64_t R, int s, int G) { return R > s ? (R - s + G - 1) / G : 0; }   // rows j of shard s with j*G+s < R

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

// ------------------------------------------------------------------------------------------------------------ redeal
int64_t RedealPlan::j0(int64_t k) const { return ceil_rows(std::min(n_live, first + k * window_rows), s, G); }

void redeal_plan(const uint32_t* h_alive, int G, int s, int64_t words, int64_t n_rows, const int64_t* toff, bool has_xh, int dpad,
                 int64_t window_rows, RedealPlan& p, cudaStream_t st)
{
    p.G = G; p.s = s; p.words = words; p.n_rows = n_rows; p.window_rows = window_rows;
    p.row_bytes = REDEAL_HEAD_BYTES + (int64_t)dpad * (int64_t)sizeof(float) + (has_xh ? (int64_t)dpad * (int64_t)sizeof(uint16_t) : 0);
    const int64_t all_words = (int64_t)G * words;
    DevArray<uint32_t> alive;
    DevArray<int64_t> cnt, wscan;
    DevArray<unsigned long long> first;
    alive.alloc(all_words > 0 ? all_words : 1);
    cnt.alloc(all_words + 1);
    wscan.alloc(all_words + 1);
    first.alloc(1);
    if (all_words > 0) KRAG_CUDA(cudaMemcpyAsync(alive.p, h_alive, sizeof(uint32_t) * (size_t)all_words, cudaMemcpyHostToDevice, st));
    word_popc_kernel<<<grid_for(all_words + 1), 256, 0, st>>>(alive.p, all_words, all_words * 32, cnt.p);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    exclusive_sum(cnt.p, wscan.p, all_words + 1, st);
    const unsigned long long none = (unsigned long long)(all_words * 32);
    KRAG_CUDA(cudaMemcpyAsync(first.p, &none, sizeof none, cudaMemcpyHostToDevice, st));
    first_dead_kernel<<<grid_for(all_words), 256, 0, st>>>(alive.p, G, words, first.p);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    unsigned long long h_first = 0;
    KRAG_CUDA(cudaMemcpyAsync(&h_first, first.p, sizeof h_first, cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaMemcpyAsync(&p.n_live, wscan.p + all_words, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    p.first = std::min<int64_t>((int64_t)h_first, p.n_live);
    p.n_windows = p.n_live > p.first ? (p.n_live - p.first + window_rows - 1) / window_rows : 0;
    p.n_new = ceil_rows(p.n_live, s, G);
    p.j_first = ceil_rows(p.first, s, G);
    const int64_t WG = p.n_windows * G;
    if (WG >= (int64_t)REDEAL_STAY) throw std::invalid_argument("too many redeal windows: raise the window width");

    DevArray<unsigned long long> tab;
    tab.alloc(3 * WG + 1);
    KRAG_CUDA(cudaMemsetAsync(tab.p, 0, sizeof(unsigned long long) * (size_t)(3 * WG + 1), st));
    DevArray<uint32_t> key, iota;
    const int64_t nr1 = n_rows > 0 ? n_rows : 1;
    key.alloc(nr1);
    iota.alloc(nr1);
    p.rank.alloc(nr1);
    redeal_rank_kernel<<<grid_for(all_words * 32), 256, 0, st>>>(alive.p, wscan.p, G, s, words, p.first, window_rows, toff, key.p, p.rank.p,
                                                                 iota.p, n_rows, tab.p, tab.p + WG, tab.p + 2 * WG);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    std::vector<unsigned long long> h_tab((size_t)(3 * WG));
    if (WG > 0) KRAG_CUDA(cudaMemcpyAsync(h_tab.data(), tab.p, sizeof(unsigned long long) * (size_t)(3 * WG), cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    p.send_rows.assign(h_tab.begin(), h_tab.begin() + WG);
    p.send_ents.assign(h_tab.begin() + WG, h_tab.begin() + 2 * WG);
    p.recv_rows.assign(h_tab.begin() + 2 * WG, h_tab.end());
    p.seg_row.assign((size_t)WG + 1, 0);
    std::vector<int64_t> seg_ent((size_t)WG + 1, 0);
    for (int64_t i = 0; i < WG; ++i) {
        p.seg_row[(size_t)i + 1] = p.seg_row[(size_t)i] + p.send_rows[(size_t)i];
        seg_ent[(size_t)i + 1] = seg_ent[(size_t)i] + p.send_ents[(size_t)i];
    }
    p.n_send = p.seg_row[(size_t)WG];

    // send order: a stable sort by (window, destination) keeps ascending rank inside each segment; the moving rows come first
    p.send_key.alloc(nr1);
    p.send_row.alloc(nr1);
    if (n_rows > 0) {
        size_t bytes = 0;
        KRAG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, key.p, p.send_key.p, iota.p, p.send_row.p, n_rows, 0, 32, st));
        DevArray<unsigned char> tmp;
        tmp.alloc(bytes ? (int64_t)bytes : 1);
        KRAG_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, key.p, p.send_key.p, iota.p, p.send_row.p, n_rows, 0, 32, st));
        count_launch();
    }
    p.send_ent.alloc(p.n_send + 1);
    if (toff) {
        DevArray<int64_t> len;
        len.alloc(p.n_send + 1);
        new_len_kernel<<<grid_for(p.n_send + 1), 256, 0, st>>>(toff, p.send_row.p, p.n_send, len.p);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        exclusive_sum(len.p, p.send_ent.p, p.n_send + 1, st);
    } else {
        KRAG_CUDA(cudaMemsetAsync(p.send_ent.p, 0, sizeof(int64_t) * (size_t)(p.n_send + 1), st));
    }
    p.seg_ent.alloc(WG + 1);
    KRAG_CUDA(cudaMemcpyAsync(p.seg_ent.p, seg_ent.data(), sizeof(int64_t) * (size_t)(WG + 1), cudaMemcpyHostToDevice, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    for (int64_t k = 0; k < p.n_windows; ++k) {   // each window's new ordinals of this shard arrive exactly once
        int64_t got = 0;
        for (int t = 0; t < G; ++t) got += p.recv_rows[(size_t)(k * G + t)];
        if (got != p.j0(k + 1) - p.j0(k)) throw std::logic_error("redeal plan: the received rows do not cover the window");
    }
}

void redeal_prepare(const int64_t* recv_ents, const int64_t* toff, const uint32_t* tid, const uint16_t* ttf, RedealPlan& p,
                    cudaStream_t st)
{
    const int G = p.G;
    const int64_t W = p.n_windows;
    p.recv_ents.assign(recv_ents, recv_ents + W * G);
    std::vector<int64_t> row_disp((size_t)(W * (G + 1))), ent_disp((size_t)(W * G));
    p.ent_base.assign((size_t)W + 1, 0);
    if (toff && p.j_first > 0) KRAG_CUDA(cudaMemcpyAsync(&p.ent_base[0], toff + p.j_first, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    int64_t max_rows = 1;
    for (int64_t k = 0; k < W; ++k) {
        int64_t r = 0, e = 0;
        for (int t = 0; t < G; ++t) {
            row_disp[(size_t)(k * (G + 1) + t)] = r;
            ent_disp[(size_t)(k * G + t)] = e;
            r += p.recv_rows[(size_t)(k * G + t)];
            e += p.recv_ents[(size_t)(k * G + t)];
        }
        row_disp[(size_t)(k * (G + 1) + G)] = r;
        p.ent_base[(size_t)k + 1] = p.ent_base[(size_t)k] + e;
        max_rows = std::max(max_rows, r);
    }
    const int64_t nnz = p.ent_base[(size_t)W];
    p.recv_row_disp.alloc(W * (G + 1) + 1);
    p.recv_ent_disp.alloc(W * G + 1);
    p.lens.alloc(max_rows);
    p.toff_new.alloc(p.n_new + 1);
    p.tid_new.alloc(nnz > 0 ? nnz : 1);
    p.ttf_new.alloc(nnz > 0 ? nnz : 1);
    p.scan_bytes = 0;
    KRAG_CUDA(cub::DeviceScan::ExclusiveScan(nullptr, p.scan_bytes, p.lens.p, p.toff_new.p, ::cuda::std::plus<int64_t>{}, (int64_t)0, max_rows, st));
    p.scan_tmp.alloc(p.scan_bytes ? (int64_t)p.scan_bytes : 1);
    if (W > 0) {
        KRAG_CUDA(cudaMemcpyAsync(p.recv_row_disp.p, row_disp.data(), sizeof(int64_t) * row_disp.size(), cudaMemcpyHostToDevice, st));
        KRAG_CUDA(cudaMemcpyAsync(p.recv_ent_disp.p, ent_disp.data(), sizeof(int64_t) * ent_disp.size(), cudaMemcpyHostToDevice, st));
    }
    // rows [0, j_first) keep their place and their term lists: copied to the new arrays as they are
    if (toff) {
        KRAG_CUDA(cudaMemcpyAsync(p.toff_new.p, toff, sizeof(int64_t) * (size_t)(p.j_first + 1), cudaMemcpyDeviceToDevice, st));
        if (p.ent_base[0] > 0) {
            KRAG_CUDA(cudaMemcpyAsync(p.tid_new.p, tid, sizeof(uint32_t) * (size_t)p.ent_base[0], cudaMemcpyDeviceToDevice, st));
            KRAG_CUDA(cudaMemcpyAsync(p.ttf_new.p, ttf, sizeof(uint16_t) * (size_t)p.ent_base[0], cudaMemcpyDeviceToDevice, st));
        }
    } else {
        KRAG_CUDA(cudaMemsetAsync(p.toff_new.p, 0, sizeof(int64_t) * (size_t)(p.j_first + 1), st));
    }
    KRAG_CUDA(cudaMemcpyAsync(p.toff_new.p + p.n_new, &p.ent_base[(size_t)W], sizeof(int64_t), cudaMemcpyHostToDevice, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
}

void redeal_pack(const RedealRows& v, const RedealPlan& p, int64_t k, void* rows, void* ents, cudaStream_t st)
{
    const int64_t p0 = p.seg_row[(size_t)(k * p.G)], n = p.seg_row[(size_t)((k + 1) * p.G)] - p0;
    if (n == 0) return;
    redeal_pack_kernel<<<grid_for(n * 32), 256, 0, st>>>(v, p.send_row.p, p.send_key.p, p.rank.p, p.send_ent.p, p.seg_ent.p, p.G, p0, n,
                                                         p.row_bytes / 16, static_cast<uint4*>(rows), static_cast<uint2*>(ents));
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

void redeal_unpack(const RedealRows& v, RedealPlan& p, int64_t k, const void* rows, const void* ents, cudaStream_t st)
{
    const int64_t j0 = p.j0(k), n = p.j0(k + 1) - j0;
    if (n == 0) return;
    const uint4* in = static_cast<const uint4*>(rows);
    redeal_unpack_rows_kernel<<<grid_for(n * 32), 256, 0, st>>>(v, in, n, p.row_bytes / 16, j0, p.lens.p);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    if (!v.dlen) return;
    size_t bytes = p.scan_bytes;
    KRAG_CUDA(cub::DeviceScan::ExclusiveScan(p.scan_tmp.p, bytes, p.lens.p, p.toff_new.p + j0, ::cuda::std::plus<int64_t>{}, p.ent_base[(size_t)k], n, st));
    count_launch();
    redeal_unpack_terms_kernel<<<grid_for(n * 32), 256, 0, st>>>(in, n, p.row_bytes / 16, static_cast<const uint2*>(ents),
                                                                 p.recv_row_disp.p + k * (p.G + 1), p.recv_ent_disp.p + k * p.G, p.G,
                                                                 p.toff_new.p, p.tid_new.p, p.ttf_new.p);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

}  // namespace krag
