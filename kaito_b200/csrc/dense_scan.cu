// dense_scan.cu -- K1: exact fp32 squared-L2 scan of the resident corpus with a fused
// top-P select.  Replaces faiss IndexIDMap(IndexFlatL2).search for small batches
// (reference call site presets/ragengine/vector_store/faiss_store.py:44-49, reached from
// vector_store/retriever/hybrid_retriever.py:209-213).
//
// HBM-bound: every corpus byte is read exactly once per pass (algorithmic bytes per pass
// = n_rows * dpad * 4); up to 4 queries share one pass.  The fp32 operation order is the
// one oracle/krag_oracle.c:l2sq_row specifies, so distances are bit-identical to it:
//   8 lanes per row, lane l owns elements {32 i + 4 l + c}: partial[c] += (x-q)^2 (FFMA),
//   s_l = (p0+p1)+(p2+p3), then an xor-butterfly over lanes 4,2,1.
//
// Layout: X row-major [n_rows, dpad], dpad % 32 == 0, zero padded.  A warp reads 8 rows
// per iteration as 2 x (4 rows x 128 contiguous bytes) per load instruction -- fully
// coalesced 128-byte segments, streamed with L1 no-allocate.  On split rows (split_rows.cuh)
// a lane reads the 16-byte high-half and low-half words of its 8 elements of a 64-element
// block (its steps 2 b and 2 b + 1: again 4 rows x 128 contiguous bytes per load) and
// rebuilds the same fp32 values.
#include "engine.h"
#include "select.cuh"
#include "split_rows.cuh"

namespace krag {

constexpr int DS_THREADS = 256;
constexpr int DS_WARPS = DS_THREADS / 32;
constexpr int DS_ROWS_PER_WARP = 8;
constexpr int DS_TILE_ROWS = DS_WARPS * DS_ROWS_PER_WARP;  // 64 rows per CTA iteration

template <int NQ, bool SPLIT>
__global__ void __launch_bounds__(DS_THREADS, 2)
dense_scan_kernel(const float* __restrict__ X, int64_t n_rows, int dpad, const uint32_t* __restrict__ alive,
                  const float* __restrict__ Q, int P, int cap, int epoch_iters, OrdMap ord_base,
                  uint64_t* __restrict__ part /*[NQ][gridDim.x][P]*/, unsigned long long* __restrict__ g_thr /*[NQ]*/)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* sq = reinterpret_cast<float*>(smem_raw);                                   // [NQ][dpad]
    uint64_t* sbuf = reinterpret_cast<uint64_t*>(smem_raw + (size_t)NQ * dpad * 4);   // [NQ][cap]
    __shared__ int s_count[NQ];
    __shared__ uint64_t s_thr[NQ];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, l8 = lane & 7, rs = lane >> 3;
    for (int i = tid; i < NQ * dpad; i += DS_THREADS) sq[i] = Q[i];
    SelectBuf sel[NQ];
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        sel[q] = SelectBuf{sbuf + (size_t)q * cap, &s_count[q], &s_thr[q], cap};
        select_init(sel[q], tid);
    }
    __syncthreads();

    const int64_t n_tiles = (n_rows + DS_TILE_ROWS - 1) / DS_TILE_ROWS;
    const int iters = (int)((n_tiles + gridDim.x - 1) / gridDim.x);
    const int steps = dpad / KRAG_LANES;
    uint64_t thr[NQ];
#pragma unroll
    for (int q = 0; q < NQ; ++q) thr[q] = KEY_PAD;

    for (int it = 0; it < iters; ++it) {
        const int64_t tile = (int64_t)it * gridDim.x + blockIdx.x;
        const int64_t rowA = tile * DS_TILE_ROWS + warp * DS_ROWS_PER_WARP + rs;
        const int64_t rowB = rowA + 4;
        const int64_t ra = rowA < n_rows ? rowA : n_rows - 1;  // clamp the address, discard the value
        const int64_t rb = rowB < n_rows ? rowB : n_rows - 1;
        const float* xa = X + ra * dpad;
        const float* xb = X + rb * dpad;
        const float4* pa = reinterpret_cast<const float4*>(xa) + l8;
        const float4* pb = reinterpret_cast<const float4*>(xb) + l8;

        float4 accA[NQ], accB[NQ];
#pragma unroll
        for (int q = 0; q < NQ; ++q) { accA[q] = make_float4(0.f, 0.f, 0.f, 0.f); accB[q] = accA[q]; }
        auto step = [&](int i, const float4& a, const float4& b) {
#pragma unroll
            for (int q = 0; q < NQ; ++q) {
                const float4 qv = *reinterpret_cast<const float4*>(sq + q * dpad + i * KRAG_LANES + l8 * 4);
                float t;
                t = a.x - qv.x; accA[q].x = fmaf(t, t, accA[q].x);
                t = a.y - qv.y; accA[q].y = fmaf(t, t, accA[q].y);
                t = a.z - qv.z; accA[q].z = fmaf(t, t, accA[q].z);
                t = a.w - qv.w; accA[q].w = fmaf(t, t, accA[q].w);
                t = b.x - qv.x; accB[q].x = fmaf(t, t, accB[q].x);
                t = b.y - qv.y; accB[q].y = fmaf(t, t, accB[q].y);
                t = b.z - qv.z; accB[q].z = fmaf(t, t, accB[q].z);
                t = b.w - qv.w; accB[q].w = fmaf(t, t, accB[q].w);
            }
        };

        if (SPLIT) {   // steps 2 b and 2 b + 1 from block b, in the same order
#pragma unroll 2
            for (int blk = 0; blk < steps / 2; ++blk) {
                float4 a0, a1, b0, b1;
                split_ld8<true>(xa, blk, l8, a0, a1);
                split_ld8<true>(xb, blk, l8, b0, b1);
                step(2 * blk, a0, b0);
                step(2 * blk + 1, a1, b1);
            }
        } else {
#pragma unroll 4
            for (int i = 0; i < steps; ++i) step(i, ldg_stream_f4(pa + i * 8), ldg_stream_f4(pb + i * 8));
        }
        const bool okA = rowA < n_rows && (alive == nullptr || bit_test(alive, (uint32_t)rowA));
        const bool okB = rowB < n_rows && (alive == nullptr || bit_test(alive, (uint32_t)rowB));
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
            float sa = (accA[q].x + accA[q].y) + (accA[q].z + accA[q].w);
            float sb = (accB[q].x + accB[q].y) + (accB[q].z + accB[q].w);
            sa += __shfl_xor_sync(0xffffffffu, sa, 4); sb += __shfl_xor_sync(0xffffffffu, sb, 4);
            sa += __shfl_xor_sync(0xffffffffu, sa, 2); sb += __shfl_xor_sync(0xffffffffu, sb, 2);
            sa += __shfl_xor_sync(0xffffffffu, sa, 1); sb += __shfl_xor_sync(0xffffffffu, sb, 1);
            if (l8 == 0) {
                if (okA) select_push(sel[q], make_key_asc(sa, ord_base + (uint32_t)rowA), thr[q]);
                if (okB) select_push(sel[q], make_key_asc(sb, ord_base + (uint32_t)rowB), thr[q]);
            }
        }
        // epoch boundary: prune lazily, only when the next epoch could overflow the buffer
        if ((it + 1) % epoch_iters == 0 && it + 1 < iters) {
            __syncthreads();
#pragma unroll
            for (int q = 0; q < NQ; ++q) {
                if (*sel[q].count + epoch_iters * DS_TILE_ROWS > cap) {
                    select_prune<DS_THREADS>(sel[q], P, tid, 0);
                    // publish this CTA's P-th best: an upper bound of the global P-th best for everyone
                    if (tid == 0 && *sel[q].count == P) atomicMin(&g_thr[q], (unsigned long long)sel[q].buf[P - 1]);
                }
                const unsigned long long h = __ldcg(&g_thr[q]);
                thr[q] = *sel[q].thr;
                if (h != KEY_PAD && h + 1 < thr[q]) thr[q] = h + 1;   // admit keys <= hint only
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        select_prune<DS_THREADS>(sel[q], P, tid, 0);
        select_store<DS_THREADS>(sel[q], P, part + ((size_t)q * gridDim.x + blockIdx.x) * P, tid);
        if (tid == 0 && *sel[q].count == P) atomicMin(&g_thr[q], (unsigned long long)sel[q].buf[P - 1]);
    }
}

static int ds_cap(int P) { return P <= 512 ? 1024 : 2048; }
static int ds_grid(const DeviceInfo& di, int64_t n_rows)
{
    int64_t n_tiles = (n_rows + DS_TILE_ROWS - 1) / DS_TILE_ROWS;
    int64_t g = 2LL * di.sm_count;  // 2 resident CTAs per SM (launch bounds), one wave, persistent
    return (int)(n_tiles < g ? (n_tiles > 0 ? n_tiles : 1) : g);
}

size_t dense_scan_part_elems(const DeviceInfo& di, int P) { return (size_t)4 * 2 * di.sm_count * P + 4; }

template <int NQ, bool SPLIT>
static void ds_launch(const DeviceInfo& di, const float* X, int64_t n_rows, int dpad, const uint32_t* alive,
                      const float* q, int P, OrdMap ord_base, uint64_t* part, unsigned long long* g_thr, cudaStream_t st)
{
    const int cap = ds_cap(P);
    const int epoch = (cap - P) / DS_TILE_ROWS > 0 ? (cap - P) / DS_TILE_ROWS : 1;
    const size_t smem = (size_t)NQ * dpad * 4 + (size_t)NQ * cap * 8;
    static bool attr_set = false;
    if (!attr_set) {
        KRAG_CUDA(cudaFuncSetAttribute(dense_scan_kernel<NQ, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        attr_set = true;
    }
    const int grid = ds_grid(di, n_rows);
    KRAG_CUDA(cudaMemsetAsync(g_thr, 0xFF, sizeof(unsigned long long) * NQ, st));
    dense_timer_begin(st, 1, n_rows * (int64_t)dpad * 4, 3 * (int64_t)NQ * n_rows * dpad);
    dense_scan_kernel<NQ, SPLIT><<<grid, DS_THREADS, smem, st>>>(X, n_rows, dpad, alive, q, P, cap, epoch, ord_base, part, g_thr);
    dense_timer_end(st);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// device rows X (split rows when split), or one staged chunk of host rows
static void scan_rows(const DeviceInfo& di, const float* X, int64_t n_rows, int dpad, const uint32_t* alive, const float* q,
                      int batch, int P, OrdMap ord_base, uint64_t* part, uint64_t* keys_out, cudaStream_t st, bool split)
{
    const int grid = ds_grid(di, n_rows);
    unsigned long long* g_thr = reinterpret_cast<unsigned long long*>(part + (size_t)4 * 2 * di.sm_count * P);
    int b = 0;
    while (b < batch) {
        int nq = batch - b >= 4 ? 4 : (batch - b >= 2 ? 2 : 1);
        // smem budget: NQ * (dpad*4 + cap*8) must stay under 100 KB (2 CTAs per SM)
        while (nq > 1 && (size_t)nq * ((size_t)dpad * 4 + (size_t)ds_cap(P) * 8) > 96 * 1024) nq >>= 1;
        const float* qb = q + (size_t)b * dpad;
        (split ? (nq == 4 ? ds_launch<4, true> : nq == 2 ? ds_launch<2, true> : ds_launch<1, true>)
               : (nq == 4 ? ds_launch<4, false> : nq == 2 ? ds_launch<2, false> : ds_launch<1, false>))(
            di, X, n_rows, dpad, alive, qb, P, ord_base, part, g_thr, st);
        // part is [nq][grid][P]: lists = CTAs
        launch_merge(part, grid, P, nq, P, /*list_stride=*/P, /*batch_stride=*/(int64_t)grid * P,
                     keys_out + (size_t)b * P, st, reinterpret_cast<const uint64_t*>(g_thr));
        b += nq;
    }
}

// chunks of the streamed scan: up to 64 MB or 64K rows, a multiple of 32 rows so a chunk's tombstone words start on a word
int64_t stream_scan_chunk_rows(int dpad)
{
    int64_t r = ((int64_t)64 << 20) / ((int64_t)dpad * 4);
    if (r > 65536) r = 65536;
    return r / 32 * 32;
}

// host rows, chunk by chunk through the staging buffers of sg
static void scan_streamed(const DeviceInfo& di, const float* X_host, int64_t n_rows, int dpad, const uint32_t* alive,
                          const float* q, int batch, int P, OrdMap ord_base, uint64_t* part, const ScanStaging& sg,
                          uint64_t* keys_out, cudaStream_t st)
{
    const int64_t R = sg.chunk_rows;
    const int64_t list = (int64_t)batch * P;
    uint64_t* run = sg.fold;            // running top P
    uint64_t* chk = sg.fold + list;     // this chunk's top P
    // the staging buffers are free once the work already queued on st is done
    KRAG_CUDA(cudaEventRecord(sg.freed[0], st));
    KRAG_CUDA(cudaEventRecord(sg.freed[1], st));
    int64_t i = 0;
    for (int64_t r0 = 0; r0 < n_rows; r0 += R, ++i) {
        const int b = (int)(i & 1);
        const int64_t m = n_rows - r0 < R ? n_rows - r0 : R;
        KRAG_CUDA(cudaStreamWaitEvent(sg.copy, sg.freed[b], 0));
        KRAG_CUDA(cudaMemcpyAsync(sg.buf[b], X_host + r0 * dpad, sizeof(float) * (size_t)(m * dpad), cudaMemcpyHostToDevice, sg.copy));
        KRAG_CUDA(cudaEventRecord(sg.copied[b], sg.copy));
        KRAG_CUDA(cudaStreamWaitEvent(st, sg.copied[b], 0));
        const OrdMap om{ord_base + (uint32_t)r0, ord_base.stride};
        scan_rows(di, sg.buf[b], m, dpad, alive ? alive + r0 / 32 : nullptr, q, batch, P, om, part, i == 0 ? run : chk, st, false);
        KRAG_CUDA(cudaEventRecord(sg.freed[b], st));
        if (i > 0) {
            launch_merge(run, 2, P, batch, P, list, P, keys_out, st);
            if (r0 + R < n_rows) KRAG_CUDA(cudaMemcpyAsync(run, keys_out, sizeof(uint64_t) * (size_t)list, cudaMemcpyDeviceToDevice, st));
        }
    }
    if (i == 1) KRAG_CUDA(cudaMemcpyAsync(keys_out, run, sizeof(uint64_t) * (size_t)list, cudaMemcpyDeviceToDevice, st));
}

void launch_dense_scan(const DeviceInfo& di, const DenseRows& rows, const uint32_t* alive, const float* q, int batch, int P,
                       OrdMap ord_base, uint64_t* part, uint64_t* keys_out, cudaStream_t st, const ScanStaging* sg)
{
    if (rows.host()) scan_streamed(di, rows.host_h(), rows.n, rows.dpad, alive, q, batch, P, ord_base, part, *sg, keys_out, st);
    else scan_rows(di, rows.dev(), rows.n, rows.dpad, alive, q, batch, P, ord_base, part, keys_out, st, rows.split());
}

}  // namespace krag
