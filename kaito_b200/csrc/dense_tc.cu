// dense_tc.cu -- K2: batched dense search on the Hopper tensor cores (wgmma).
//
// Replaces faiss IndexFlatL2.search for query batches (its nq >= 20 sgemm path; reference
// call site presets/ragengine/vector_store/faiss_store.py:44-49 via hybrid_retriever.py:209-213).
//
//   1. the prune pass (wgmma, TMA-staged, accumulators in registers): D[corpus rows x NQ queries] = X_tile . Q^T
//        dense_tc_bf16_kernel<NQ, DUMP>  192-row tiles, bf16 corpus and queries from shared memory: 2 bytes/element from
//                   HBM.  The corpus operand is the high halves of split rows (split_rows.cuh: the default on rows with
//                   dpad % 64 == 0), the opt-in bf16 shadow (KRAG_DENSE_TC_BF16) or the device copy of host-resident rows
//        dense_tc_kernel<NQ, MODE, DUMP>  128-row tiles, fp32 operands consumed as TF32:
//          TC_TF32  plain fp32 corpus rows and queries straight from shared memory
//          TC_TF32S TC_TF32 on split rows: both halves staged by TMA, rebuilt to fp32 in the A registers (tf32 wgmma with A
//                   from registers); the same products as TC_TF32 on the plain rows, bit for bit
//        epilogue: a = |x|^2 - 2 x.q  per (row, query), compared with a per-query threshold;
//        rows below it are appended to that query's candidate list (rare: ~C of N rows).
//        DUMP mode writes `a` for a strided 1/64 sample of the tiles instead.
//   2. sample_threshold_kernel: per query, the m-th smallest sampled `a` -> threshold that
//        admits ~C = max(512, 4P) rows of the full corpus.
//   3. rescore_kernel: EXACT fp32 squared L2 of every candidate in K1's operation order
//        (bit-identical to dense_scan.cu / the oracle), then the ordinary top-P merge.
//   4. certify_kernel: a query's result is exact if every non-candidate row is provably
//        farther than the P-th exact distance:  D_P <= thr + |q|^2 - 2 eps,  eps = worst-case
//        dot-product error of the main pass times |x|_max |q|.  Queries that fail (candidate
//        overflow, adversarial near-duplicates) are re-run on the exact scan kernel K1.
//
// So the tensor cores only PRUNE; every returned score is an exact fp32 distance.
//
// Roofline: bytes = n_rows*dpad*2 per bf16 pass, n_rows*dpad*4 per tf32 pass (HBM), flops = 2*NQ*n_rows*dpad.  Every
// tile also stages all NQ query rows from L2 into shared memory: NQ / tile rows query bytes per corpus byte (bf16 pass).
#include <cuda.h>
#include <cuda_bf16.h>
#include <math_constants.h>

#include <atomic>
#include <mutex>
#include <vector>

#include "engine.h"
#include "select.cuh"
#include "split_rows.cuh"
#include "tc_ptx.cuh"

namespace krag {

// ------------------------------------------------------------------------- the kernel
constexpr int TC_TILE_M = 128;          // corpus rows per TF32 tile: two consumer warpgroups x wgmma M = 64
constexpr int TC_KBLOCK = 32;           // fp32 elements per k-block = one 128-byte swizzle row
constexpr int TC_THREADS = 384;         // warpgroup 0: TMA producer, warpgroups 1-2: wgmma + epilogue
constexpr int TC_SAMPLE_STRIDE = 64;    // DUMP mode visits every 64th tile
constexpr int TC_A_BYTES = TC_TILE_M * 128;  // 16 KB: 128 rows x one 128-byte swizzle row (32 fp32 or 64 halves)
constexpr int TC_DUMP_GROUP = 16;       // rows per minimum in the threshold-sampling dump (one warp's wgmma rows)
constexpr int TC16_TILE_M = 192;        // corpus rows per bf16 tile: three wgmma M = 64 blocks
constexpr int TC16_THREADS = 256;       // two warpgroups, both wgmma + epilogue; thread 0 also issues the TMA loads

enum { TC_TF32 = 0, TC_TF32S = 2 };

// One ring; a stage holds the corpus rows of the tile and all NQ query rows for 32 (TF32) or 64 (TF32S) elements of the
// dimension: 4 wgmma K steps (8 in TF32S mode, whose stage holds one 64-element block of split rows: its high-half and
// low-half boxes, and two fp32 query boxes).
template <int NQ, int MODE> struct TcCfg {
    static constexpr int A_BYTES = (MODE == TC_TF32S ? 2 : 1) * TC_A_BYTES;
    static constexpr int Q_BYTES = (MODE == TC_TF32S ? 2 : 1) * NQ * 128;
    static constexpr int STAGE_BYTES = A_BYTES + Q_BYTES;
    static constexpr int STAGES = (200 * 1024) / STAGE_BYTES > 8 ? 8 : (200 * 1024) / STAGE_BYTES;
    static constexpr int ELEMS = MODE == TC_TF32 ? TC_KBLOCK : 2 * TC_KBLOCK;   // dimension elements per stage
    static constexpr int BAR_BYTES = 256;
    static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + BAR_BYTES + NQ * 4;
};
// The bf16 ring: a stage holds the 192 corpus rows of the tile and all NQ query rows for 64 elements (4 wgmma K steps).
// 4 stages of 56 KB at NQ = 256 (224 KB + barriers + thresholds: inside the 227 KB opt-in).
template <int NQ> struct Tc16Cfg {
    static constexpr int A_BYTES = TC16_TILE_M * 128;
    static constexpr int STAGE_BYTES = A_BYTES + NQ * 128;
    static constexpr int STAGES = (224 * 1024) / STAGE_BYTES > 8 ? 8 : (224 * 1024) / STAGE_BYTES;
    static constexpr int ELEMS = 2 * TC_KBLOCK;
    static constexpr int BAR_BYTES = 256;
    static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + BAR_BYTES + NQ * 4;
};

// tf32 A fragment (mma.sync m16n8k8 / wgmma register layout) of K step s (0..7) from a TF32S stage: the high-half box at
// `hi`, the low-half box TC_A_BYTES later, each 128 rows x 64 halves (a block's half in split_pos order), 128B-swizzled.
// This thread's rows r and r + 8 (r & 7 == g), elements e = 8 s + q and e + 4, gathered in element order and rebuilt to
// their fp32 bits:  a0 (r, e), a1 (r + 8, e), a2 (r, e + 4), a3 (r + 8, e + 4).
__device__ __forceinline__ void tf32s_a_fragment(const unsigned char* hi, int r, int g, int q, int s, uint32_t* a)
{
    const unsigned char* lo = hi + TC_A_BYTES;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int p = split_pos(8 * s + q + 4 * (k >> 1));
        const int o = (r + 8 * (k & 1)) * 128 + (((p >> 3) ^ g) << 4) + 2 * (p & 7);
        a[k] = split_join(*reinterpret_cast<const uint16_t*>(hi + o), *reinterpret_cast<const uint16_t*>(lo + o));
    }
}

// Epilogue of one wgmma accumulator block, straight from its registers: acc[4i + 2h + c] is (tile row ra + 8h, query
// qoff + 8i + 2q + c), i < R / 4, and xn[h] that row's |x|^2 (+inf: past the end or deleted).
//   main pass: the rows with a = |x|^2 - 2 x.q below the query's threshold go to its candidate list
//   DUMP, dump_min: threshold sampling, per query only the minimum of a over this warp's 16 rows, as dump group grp
//   DUMP, !dump_min: a itself, in dump column dcol0 + row (columns from S on are not written)
template <int R, bool DUMP>
__device__ __forceinline__ void tc_epilogue(float* acc, const float* xn, int ra, int qoff, int g, int q, int64_t tile_row0,
                                            const float* s_thr, uint32_t* cand_count, uint32_t* cand_rows, int cap,
                                            float* dump, int64_t S, int dump_min, int64_t grp, int64_t dcol0)
{
    if (DUMP) {
        if (dump_min) {
            // the few smallest values of the sample, which is all the threshold needs, survive
#pragma unroll
            for (int i = 0; i < R / 4; ++i) {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float v = fminf(fmaf(-2.f, acc[4 * i + c], xn[0]), fmaf(-2.f, acc[4 * i + 2 + c], xn[1]));
                    v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 4));
                    v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 8));
                    v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 16));
                    if (g == 0) dump[(int64_t)(qoff + 8 * i + 2 * q + c) * S + grp] = v;
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < R / 4; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int c = 0; c < 2; ++c)
                        if (dcol0 + ra + 8 * h < S)
                            dump[(int64_t)(qoff + 8 * i + 2 * q + c) * S + dcol0 + ra + 8 * h] = fmaf(-2.f, acc[4 * i + 2 * h + c], xn[h]);
        }
    } else {
        // s_thr[j] = thr_j / 2 (see the kernels); ~2 instructions per (row, query) pair on the common path: one add and one max; hits are ~1 in 20000
        const float half0 = 0.5f * xn[0], half1 = 0.5f * xn[1];
        float mx0 = -CUDART_INF_F, mx1 = -CUDART_INF_F;
#pragma unroll
        for (int i = 0; i < R / 4; ++i) {
            const float2 t = *reinterpret_cast<const float2*>(s_thr + qoff + 8 * i + 2 * q);
            acc[4 * i + 0] += t.x; acc[4 * i + 1] += t.y; acc[4 * i + 2] += t.x; acc[4 * i + 3] += t.y;
            mx0 = fmaxf(mx0, fmaxf(acc[4 * i + 0], acc[4 * i + 1]));
            mx1 = fmaxf(mx1, fmaxf(acc[4 * i + 2], acc[4 * i + 3]));
        }
        if (mx0 > half0 || mx1 > half1) {   // rare: some pair passes  x.q + thr/2 > |x|^2/2
#pragma unroll
            for (int i = 0; i < R / 4; ++i) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        if (acc[4 * i + 2 * h + c] > (h ? half1 : half0)) {
                            const int j = qoff + 8 * i + 2 * q + c;
                            const uint32_t pos = atomicAdd(&cand_count[j], 1u);
                            if (pos < (uint32_t)cap) cand_rows[(size_t)j * cap + pos] = (uint32_t)(tile_row0 + ra + 8 * h);
                        }
                    }
                }
            }
        }
    }
}

template <int NQ, int MODE, bool DUMP>
__global__ void __launch_bounds__(TC_THREADS, 1)
dense_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmQ, int64_t n_rows,
                int kblocks /*stages per tile*/, int64_t n_ltiles, int tile_stride, const float* __restrict__ xnorm,
                const uint32_t* __restrict__ alive, const float* __restrict__ thr_g, uint32_t* __restrict__ cand_count,
                uint32_t* __restrict__ cand_rows, int cap, float* __restrict__ dump, int64_t S, int dump_min)
{
    using Cfg = TcCfg<NQ, MODE>;
    constexpr int R = NQ / 2;                   // accumulators per thread
    extern __shared__ unsigned char tc_smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* tail = smem + (size_t)Cfg::STAGES * Cfg::STAGE_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);            // [STAGES] producer arrival + TMA bytes
    uint64_t* empty_bar = full_bar + Cfg::STAGES;                       // [STAGES] one arrival per consumer warp
    float* s_thr = reinterpret_cast<float*>(tail + Cfg::BAR_BYTES);     // [NQ]
    static_assert(2 * Cfg::STAGES * 8 <= Cfg::BAR_BYTES, "barrier area too small");

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmQ);
        for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
        fence_barrier_init();
    }
    // s_thr[j] = thr_j / 2:  a = |x|^2 - 2 x.q < thr_j   <=>   x.q + thr_j/2 > |x|^2/2
    if (!DUMP) for (int j = threadIdx.x; j < NQ; j += TC_THREADS) s_thr[j] = 0.5f * thr_g[j];
    __syncthreads();

    if (warp < 4) {
        // ===================== producer: corpus rows (HBM stream, read once) + query rows (L2-resident) =====================
        regs_dealloc<40>();
        if (threadIdx.x == 0) {
            int stage = 0; uint32_t phase = 0;
            for (int64_t lt = blockIdx.x; lt < n_ltiles; lt += gridDim.x) {
                const int row0 = (int)(lt * tile_stride * TC_TILE_M);
                for (int kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    unsigned char* sa = smem + (size_t)stage * Cfg::STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                    if (MODE == TC_TF32S) {   // split rows: the high and the low halves of block kb, two query boxes
                        tma_load_3d(sa, &tmX, &full_bar[stage], 0, 2 * kb, row0, TMA_EVICT_FIRST);
                        tma_load_3d(sa + TC_A_BYTES, &tmX, &full_bar[stage], 0, 2 * kb + 1, row0, TMA_EVICT_FIRST);
                        tma_load_2d(sa + Cfg::A_BYTES + NQ * 128, &tmQ, &full_bar[stage], kb * Cfg::ELEMS + TC_KBLOCK, 0, TMA_EVICT_LAST);
                    } else {
                        tma_load_2d(sa, &tmX, &full_bar[stage], kb * Cfg::ELEMS, row0, TMA_EVICT_FIRST);
                    }
                    tma_load_2d(sa + Cfg::A_BYTES, &tmQ, &full_bar[stage], kb * Cfg::ELEMS, 0, TMA_EVICT_LAST);
                    if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64) =====================
        regs_alloc<232>();
        const int wg = (warp >> 2) - 1, w = warp & 3;
        const int g = lane >> 2, q = lane & 3;
        const int r_lo = 64 * wg + 16 * w + g;                 // this thread's accumulator rows: r_lo and r_lo + 8
        float acc[R];
        int stage = 0; uint32_t phase = 0;
        for (int64_t lt = blockIdx.x; lt < n_ltiles; lt += gridDim.x) {
            for (int kb = 0; kb < kblocks; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                unsigned char* sa = smem + (size_t)stage * Cfg::STAGE_BYTES;
                const uint64_t bdesc = wgmma_desc_sw128(smem_u32(sa + Cfg::A_BYTES));
                if (MODE == TC_TF32S) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {              // query box h: elements 32 h .. 32 h + 31 of the block
                        uint32_t af[4][4];
#pragma unroll
                        for (int s = 0; s < 4; ++s) tf32s_a_fragment(sa, r_lo, g, q, 4 * h + s, af[s]);
                        wgmma_fence();
#pragma unroll
                        for (int s = 0; s < 4; ++s)
                            wgmma_tf32_rs<NQ>(acc, af[s], bdesc + h * (NQ * 128 / 16) + 2 * s, (uint32_t)((kb | h | s) != 0));
                        wgmma_commit();
                        wgmma_wait<0>();                       // the A registers are reused by the next K steps
                    }
                } else {
                    const uint64_t adesc = wgmma_desc_sw128(smem_u32(sa + wg * 64 * 128));
                    wgmma_fence();
#pragma unroll
                    for (int s = 0; s < 4; ++s)                // K steps of 32 bytes: 8 tf32
                        wgmma_tf32_ss<NQ>(acc, adesc + 2 * s, bdesc + 2 * s, (uint32_t)((kb | s) != 0));
                    wgmma_commit();
                    wgmma_wait<0>();
                }
                wgmma_fence_operands<R>(acc);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[stage]);
                if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
            }
            // ===================== epilogue straight from the accumulator registers =====================
            // acc[4i + 2h + c] is (row r_lo + 8h, query 8i + 2q + c)
            const int64_t tile_row0 = lt * tile_stride * TC_TILE_M;
            float xn[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = tile_row0 + r_lo + 8 * h;
                xn[h] = CUDART_INF_F;
                if (row < n_rows && (alive == nullptr || bit_test(alive, (uint32_t)row))) xn[h] = xnorm[row];
            }
            tc_epilogue<R, DUMP>(acc, xn, r_lo, 0, g, q, tile_row0, s_thr, cand_count, cand_rows, cap, dump, S, dump_min,
                                 lt * (TC_TILE_M / TC_DUMP_GROUP) + 4 * wg + w, lt * TC_TILE_M);
        }
    }
}

// The bf16 prune pass on 192-row tiles.  A stage's query rows come from L2 once per tile, so a taller tile reads fewer
// query bytes per corpus byte: NQ / 192 instead of NQ / 128.  The accumulators bound the tile: 192 x NQ fp32 over 256
// threads is 3 NQ / 4 registers per thread, which leaves no registers for a separate producer warp (ptxas holds every
// thread of the kernel to 65536 / threads, whatever setmaxnreg says).  So both warpgroups compute:
//   warpgroup wg: tile rows [64 wg, 64 wg + 64) x all NQ queries                (m64nNQ,     acc0: NQ / 2 per thread)
//                 tile rows [128, 192)         x queries [wg NQ/2, wg NQ/2 + NQ/2) (m64n(NQ/2), acc1: NQ / 4 per thread)
// and thread 0 issues the TMA loads, across tile boundaries.  One wgmma group stays in flight: a warp releases the stage of
// k-block i - 1 once it has issued k-block i's group and group i - 1 has completed, and thread 0 then refills that stage
// with k-block i - 1 + STAGES.  This cannot deadlock: thread 0 waits on `empty` only for a stage its own warp has already
// released, and the other warps' releases of k-block i - 1 need only `full` of k-block i, loaded before, never further
// progress of thread 0.  Every (row, query) product is the same wgmma k16 sequence as a 128-row tile's: the same operands
// in the same order.
template <int NQ, bool DUMP>
__global__ void __launch_bounds__(TC16_THREADS, 1)
dense_tc_bf16_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmQ, int64_t n_rows,
                     int kblocks /*stages per tile*/, int piece_step /*128-byte pieces per k-block*/, int64_t n_ltiles,
                     int row_step /*first rows of consecutive tiles*/, const float* __restrict__ xnorm, const uint32_t* __restrict__ alive,
                     const float* __restrict__ thr_g, uint32_t* __restrict__ cand_count, uint32_t* __restrict__ cand_rows,
                     int cap, float* __restrict__ dump, int64_t S, int dump_min)
{
    using Cfg = Tc16Cfg<NQ>;
    constexpr int R0 = NQ / 2, R1 = NQ / 4;    // accumulators per thread: the warpgroup's own 64 rows, the shared 64 rows
    extern __shared__ unsigned char tc_smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* tail = smem + (size_t)Cfg::STAGES * Cfg::STAGE_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);            // [STAGES] producer arrival + TMA bytes
    uint64_t* empty_bar = full_bar + Cfg::STAGES;                       // [STAGES] one arrival per warp
    float* s_thr = reinterpret_cast<float*>(tail + Cfg::BAR_BYTES);     // [NQ]
    static_assert(2 * Cfg::STAGES * 8 <= Cfg::BAR_BYTES, "barrier area too small");

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2, w = warp & 3, g = lane >> 2, q = lane & 3;
    const int r0 = 64 * wg + 16 * w + g;        // acc0 rows r0, r0 + 8
    const int r1 = 128 + 16 * w + g;            // acc1 rows r1, r1 + 8
    const int q1 = wg * (NQ / 2);               // acc1's first query

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmQ);
        for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
        fence_barrier_init();
    }
    // s_thr[j] = thr_j / 2:  a = |x|^2 - 2 x.q < thr_j   <=>   x.q + thr_j/2 > |x|^2/2
    if (!DUMP) for (int j = threadIdx.x; j < NQ; j += TC16_THREADS) s_thr[j] = 0.5f * thr_g[j];
    __syncthreads();

    // producer state (thread 0): the next k-block to load, flattened over this CTA's tiles
    int64_t p_lt = blockIdx.x;
    int p_kb = 0, p_stage = 0;
    uint32_t p_phase = 0;
    auto produce = [&]() {
        if (p_lt >= n_ltiles) return;
        mbar_wait(&empty_bar[p_stage], p_phase ^ 1);
        unsigned char* sa = smem + (size_t)p_stage * Cfg::STAGE_BYTES;
        mbar_expect_tx(&full_bar[p_stage], Cfg::STAGE_BYTES);
        tma_load_3d(sa, &tmX, &full_bar[p_stage], 0, p_kb * piece_step, (int)(p_lt * row_step), TMA_EVICT_FIRST);
        tma_load_2d(sa + Cfg::A_BYTES, &tmQ, &full_bar[p_stage], p_kb * Cfg::ELEMS, 0, TMA_EVICT_LAST);
        if (++p_stage == Cfg::STAGES) { p_stage = 0; p_phase ^= 1; }
        if (++p_kb == kblocks) { p_kb = 0; p_lt += gridDim.x; }
    };
    if (threadIdx.x == 0)
        for (int i = 0; i < Cfg::STAGES; ++i) produce();
    // this warp is done with `stage`: release it, and thread 0 refills it
    auto release = [&](int stage) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (threadIdx.x == 0) produce();
        __syncwarp();
    };

    float acc0[R0], acc1[R1];
    int stage = 0, prev = 0; uint32_t phase = 0;
    for (int64_t lt = blockIdx.x; lt < n_ltiles; lt += gridDim.x) {
        const int64_t tile_row0 = lt * row_step;
        float xn0[2], xn1[2];
        for (int kb = 0; kb < kblocks; ++kb) {
            if (kb == kblocks - 1) {   // the epilogue's row norms, loaded while the last k-block lands and multiplies
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t ra = tile_row0 + r0 + 8 * h, rb = tile_row0 + r1 + 8 * h;
                    xn0[h] = (ra < n_rows && (alive == nullptr || bit_test(alive, (uint32_t)ra))) ? xnorm[ra] : CUDART_INF_F;
                    xn1[h] = (rb < n_rows && (alive == nullptr || bit_test(alive, (uint32_t)rb))) ? xnorm[rb] : CUDART_INF_F;
                }
            }
            mbar_wait(&full_bar[stage], phase);
            unsigned char* sa = smem + (size_t)stage * Cfg::STAGE_BYTES;
            const uint64_t adesc0 = wgmma_desc_sw128(smem_u32(sa + wg * 64 * 128));
            const uint64_t adesc1 = wgmma_desc_sw128(smem_u32(sa + 128 * 128));
            const uint64_t bdesc0 = wgmma_desc_sw128(smem_u32(sa + Cfg::A_BYTES));
            const uint64_t bdesc1 = wgmma_desc_sw128(smem_u32(sa + Cfg::A_BYTES + q1 * 128));
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < 4; ++s) {              // K steps of 32 bytes: 16 bf16
                wgmma_bf16_ss<NQ>(acc0, adesc0 + 2 * s, bdesc0 + 2 * s, (uint32_t)((kb | s) != 0));
                wgmma_bf16_ss<NQ / 2>(acc1, adesc1 + 2 * s, bdesc1 + 2 * s, (uint32_t)((kb | s) != 0));
            }
            wgmma_commit();
            if (kb > 0) {
                wgmma_wait<1>();                       // k-block kb - 1's group is done with its stage
                release(prev);
            }
            prev = stage;
            if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_operands<R0>(acc0);
        wgmma_fence_operands<R1>(acc1);
        release(prev);
        // 12 dump groups of 16 rows per tile: 4 wg + w for acc0, 8 + w for acc1 (each warpgroup writes half its queries)
        const int64_t grp0 = lt * (TC16_TILE_M / TC_DUMP_GROUP);
        tc_epilogue<R0, DUMP>(acc0, xn0, r0, 0, g, q, tile_row0, s_thr, cand_count, cand_rows, cap, dump, S, dump_min,
                              grp0 + 4 * wg + w, tile_row0);
        tc_epilogue<R1, DUMP>(acc1, xn1, r1, q1, g, q, tile_row0, s_thr, cand_count, cand_rows, cap, dump, S, dump_min,
                              grp0 + 8 + w, tile_row0);
    }
}

// fp32 -> bf16 (round to nearest even) shadow rows; n4 = number of float4 groups
__global__ void f32_to_bf16_kernel(const float4* __restrict__ in, uint2* __restrict__ out, int64_t n4)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 v = in[i];
        const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
        uint2 o;
        o.x = *reinterpret_cast<const uint32_t*>(&a); o.y = *reinterpret_cast<const uint32_t*>(&b);
        out[i] = o;
    }
}
void launch_f32_to_bf16(const float* in, uint16_t* out, int64_t n_elems, cudaStream_t st)
{
    if (n_elems == 0) return;
    const int64_t n4 = n_elems / 4;
    int64_t blocks = (n4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    f32_to_bf16_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(in), reinterpret_cast<uint2*>(out), n4);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// host-resident rows: bf16 copy (round to nearest even, as f32_to_bf16_kernel) and r = |x - bf16(x)| rounded up, one warp per
// row.  x - bf16(x) is exact in fp32 (the two are within a factor of 2: Sterbenz), so only the sum and the root round, upwards.
__global__ void __launch_bounds__(256)
bf16_residual_kernel(const float* __restrict__ X, int64_t n, int dpad, uint16_t* __restrict__ Xh, float* __restrict__ xres)
{
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n) return;
    const float4* p = reinterpret_cast<const float4*>(X + r * dpad);
    uint2* o = reinterpret_cast<uint2*>(Xh + r * dpad);
    float s = 0.f;
    for (int i = lane; i < dpad / 4; i += 32) {
        const float4 v = p[i];
        const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
        const float e0 = v.x - __low2float(a), e1 = v.y - __high2float(a), e2 = v.z - __low2float(b), e3 = v.w - __high2float(b);
        s = __fmaf_ru(e0, e0, s); s = __fmaf_ru(e1, e1, s); s = __fmaf_ru(e2, e2, s); s = __fmaf_ru(e3, e3, s);
        uint2 w;
        w.x = *reinterpret_cast<const uint32_t*>(&a); w.y = *reinterpret_cast<const uint32_t*>(&b);
        o[i] = w;
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) s = __fadd_ru(s, __shfl_xor_sync(0xffffffffu, s, k));
    if (lane == 0) xres[r] = __fsqrt_ru(s);
}
void launch_bf16_residual(const float* X, int64_t n, int dpad, uint16_t* Xh, float* xres, cudaStream_t st)
{
    if (n == 0) return;
    bf16_residual_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(X, n, dpad, Xh, xres);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// ------------------------------------------------------------- row norms (index time)
__global__ void __launch_bounds__(256)
row_norms_kernel(const float* __restrict__ X, int64_t row0, int64_t n, int dpad, float* __restrict__ xnorm,
                 uint32_t* __restrict__ xn_max_bits)
{
    const int lane = threadIdx.x & 31;
    const int64_t r = row0 + (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (r >= row0 + n) return;
    const float4* p = reinterpret_cast<const float4*>(X + r * dpad);
    float s = 0.f;
    for (int i = lane; i < dpad / 4; i += 32) { float4 v = p[i]; s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) { xnorm[r] = s; atomicMax(xn_max_bits, __float_as_uint(s)); }
}
void launch_row_norms(const float* X, int64_t row0, int64_t n, int dpad, float* xnorm, uint32_t* xn_max_bits, cudaStream_t st)
{
    if (n == 0) return;
    row_norms_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(X, row0, n, dpad, xnorm, xn_max_bits);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// -------------------------------------------------------- sample -> per-query threshold
constexpr int ST_THREADS = 512;
// CAP = 1024 when m <= 256: the first prune (a bitonic sort of CAP keys, the dominant cost of this kernel) comes after two
// iterations instead of three and sorts half as many keys
template <int ST_CAP>
__global__ void __launch_bounds__(ST_THREADS)
sample_threshold_kernel(const float* __restrict__ dump, int64_t S, int m, int nq_valid, float* __restrict__ thr,
                        float* __restrict__ part_vals /* != null: grid (NQ, parts), write this part's m smallest values */)
{
    __shared__ uint64_t s_buf[ST_CAP];
    __shared__ int s_count;
    __shared__ uint64_t s_thr;
    const int tid = threadIdx.x, j = blockIdx.x;
    const int parts = gridDim.y, part = blockIdx.y;
    if (j >= nq_valid) {                                                    // padded query: admits nothing
        if (part_vals) { for (int i = tid; i < m; i += ST_THREADS) part_vals[((int64_t)j * parts + part) * m + i] = CUDART_INF_F; }
        else if (tid == 0) thr[j] = -CUDART_INF_F;
        return;
    }
    SelectBuf sel{s_buf, &s_count, &s_thr, ST_CAP};
    select_init(sel, tid);
    __syncthreads();
    // this block's slice of the query's samples (two-level selection: `parts` blocks per query, then one more pass
    // of this kernel over their parts * m survivors)
    const int64_t lo = S * part / parts, hi = S * (part + 1) / parts;
    const float* col = dump + (int64_t)j * S + lo;
    S = hi - lo;
    const int epoch = (ST_CAP - m) / ST_THREADS;
    uint64_t t = KEY_PAD;
    int it = 0;
    for (int64_t i0 = 0; i0 < S; i0 += ST_THREADS, ++it) {
        int64_t i = i0 + tid;
        if (i < S) select_push(sel, make_key_asc(col[i], (uint32_t)i), t);
        if ((it + 1) % epoch == 0) {
            __syncthreads();
            if (s_count + epoch * ST_THREADS > ST_CAP) select_prune<ST_THREADS>(sel, m, tid, 0);
            t = s_thr;
        }
    }
    select_prune<ST_THREADS>(sel, m, tid, 0);
    if (part_vals) {
        for (int i = tid; i < m; i += ST_THREADS)
            part_vals[((int64_t)j * parts + part) * m + i] = (i < s_count) ? key_value_asc(s_buf[i]) : CUDART_INF_F;
    } else if (tid == 0) {
        thr[j] = (s_count >= m) ? key_value_asc(s_buf[m - 1]) : CUDART_INF_F;
    }
}

// ------------------------------------------------------------------ exact rescoring
// one 8-lane group per candidate; same arithmetic as dense_scan_kernel / oracle l2sq_row, on plain or split rows
template <bool SPLIT>
__global__ void __launch_bounds__(256)
rescore_kernel(const float* __restrict__ X, int dpad, const float* __restrict__ Q, const uint32_t* __restrict__ cand_count,
               const uint32_t* __restrict__ cand_rows, int cap, OrdMap ord_base, uint64_t* __restrict__ exact_keys)
{
    extern __shared__ __align__(16) float rs_q[];   // [dpad]
    const int j = blockIdx.y, tid = threadIdx.x, lane = tid & 31, l8 = lane & 7;
    const int cnt = (int)min(cand_count[j], (uint32_t)cap);
    const int c = blockIdx.x * 32 + (tid >> 3);
    if (blockIdx.x * 32 >= cnt) {   // whole block past the end: pad and leave
        if (l8 == 0 && c < cap) exact_keys[(size_t)j * cap + c] = KEY_PAD;
        return;
    }
    for (int i = tid; i < dpad; i += 256) rs_q[i] = Q[(size_t)j * dpad + i];
    __syncthreads();
    const bool valid = c < cnt;
    const uint32_t row = valid ? cand_rows[(size_t)j * cap + c] : 0u;
    const float* xr = X + (size_t)row * dpad;
    const float4* p = reinterpret_cast<const float4*>(xr) + l8;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const int steps = dpad / KRAG_LANES;
    auto step = [&](int i, const float4& a) {
        const float4 qv = *reinterpret_cast<const float4*>(rs_q + i * KRAG_LANES + l8 * 4);
        float t;
        t = a.x - qv.x; acc.x = fmaf(t, t, acc.x);
        t = a.y - qv.y; acc.y = fmaf(t, t, acc.y);
        t = a.z - qv.z; acc.z = fmaf(t, t, acc.z);
        t = a.w - qv.w; acc.w = fmaf(t, t, acc.w);
    };
    if (SPLIT) {   // steps 2 b and 2 b + 1 from block b, in the same order
#pragma unroll 2
        for (int b = 0; b < steps / 2; ++b) {
            float4 a0, a1;
            split_ld8<false>(xr, b, l8, a0, a1);
            step(2 * b, a0);
            step(2 * b + 1, a1);
        }
    } else {
#pragma unroll 4
        for (int i = 0; i < steps; ++i) step(i, __ldg(p + i * 8));
    }
    float s = (acc.x + acc.y) + (acc.z + acc.w);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    if (l8 == 0 && c < cap) exact_keys[(size_t)j * cap + c] = valid ? make_key_asc(s, ord_base + row) : KEY_PAD;
}

// rescore_kernel's arithmetic on rows in pinned host memory, read through their mapped device address (zero-copy over the
// host link) with plain ld.global: the non-coherent path is not relied on for host-mapped memory
__global__ void __launch_bounds__(256)
rescore_mapped_kernel(const float* __restrict__ X, int dpad, const float* __restrict__ Q, const uint32_t* __restrict__ cand_count,
                      const uint32_t* __restrict__ cand_rows, int cap, OrdMap ord_base, uint64_t* __restrict__ exact_keys)
{
    extern __shared__ __align__(16) float rm_q[];   // [dpad]
    const int j = blockIdx.y, tid = threadIdx.x, lane = tid & 31, l8 = lane & 7;
    const int cnt = (int)min(cand_count[j], (uint32_t)cap);
    const int c = blockIdx.x * 32 + (tid >> 3);
    if (blockIdx.x * 32 >= cnt) {
        if (l8 == 0 && c < cap) exact_keys[(size_t)j * cap + c] = KEY_PAD;
        return;
    }
    for (int i = tid; i < dpad; i += 256) rm_q[i] = Q[(size_t)j * dpad + i];
    __syncthreads();
    const bool valid = c < cnt;
    const uint32_t row = valid ? cand_rows[(size_t)j * cap + c] : 0u;
    const float4* p = reinterpret_cast<const float4*>(X + (size_t)row * dpad) + l8;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const int steps = dpad / KRAG_LANES;
#pragma unroll 4
    for (int i = 0; i < steps; ++i) {
        float4 a;
        asm("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(a.x), "=f"(a.y), "=f"(a.z), "=f"(a.w) : "l"(p + i * 8));
        const float4 qv = *reinterpret_cast<const float4*>(rm_q + i * KRAG_LANES + l8 * 4);
        float t;
        t = a.x - qv.x; acc.x = fmaf(t, t, acc.x);
        t = a.y - qv.y; acc.y = fmaf(t, t, acc.y);
        t = a.z - qv.z; acc.z = fmaf(t, t, acc.z);
        t = a.w - qv.w; acc.w = fmaf(t, t, acc.w);
    }
    float s = (acc.x + acc.y) + (acc.z + acc.w);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    if (l8 == 0 && c < cap) exact_keys[(size_t)j * cap + c] = valid ? make_key_asc(s, ord_base + row) : KEY_PAD;
}

// ------------------------------------------------------------- refine (host-resident rows)
// For every candidate of the main pass, an interval [L, U] that holds its exact distance D = |x - q|^2, computed from the
// device bf16 copy b = bf16(x) and r >= |x - b| (xres):  |b - q| - r <= |x - q| <= |b - q| + r  (triangle inequality).
// d_lo <= |b - q|^2 <= d_hi come from directed rounding throughout (no error model needed); then
//   L = max(0, sqrt_rd(d_lo) - r)^2 rounded down,   U = (sqrt_ru(d_hi) + r)^2 rounded up.
// One 8-lane group per candidate as in rescore_kernel; lane l8 reads 8 bf16 elements (16 bytes) per 64-element step.
__device__ __forceinline__ void refine_acc(float b, float q, float& lo, float& hi)
{
    // b - q rounded both ways: both results carry the sign of the exact difference (or are zero)
    const float t_lo = __fsub_rd(b, q), t_hi = __fsub_ru(b, q);
    const float m_lo = t_lo >= 0.f ? t_lo : -t_hi, m_hi = t_lo >= 0.f ? t_hi : -t_lo;
    lo = __fmaf_rd(m_lo, m_lo, lo);
    hi = __fmaf_ru(m_hi, m_hi, hi);
}
__global__ void __launch_bounds__(256)
refine_kernel(const uint16_t* __restrict__ Xh, const float* __restrict__ xres, int dpad, const float* __restrict__ Q,
              const uint32_t* __restrict__ cand_count, const uint32_t* __restrict__ cand_rows, int cap,
              float* __restrict__ lo_out, uint64_t* __restrict__ u_keys)
{
    extern __shared__ __align__(16) float rf_q[];   // [dpad]
    const int j = blockIdx.y, tid = threadIdx.x, lane = tid & 31, l8 = lane & 7;
    const int cnt = (int)min(cand_count[j], (uint32_t)cap);
    const int c = blockIdx.x * 32 + (tid >> 3);
    if (blockIdx.x * 32 >= cnt) {
        if (l8 == 0 && c < cap) u_keys[(size_t)j * cap + c] = KEY_PAD;
        return;
    }
    for (int i = tid; i < dpad; i += 256) rf_q[i] = Q[(size_t)j * dpad + i];
    __syncthreads();
    const bool valid = c < cnt;
    const uint32_t row = valid ? cand_rows[(size_t)j * cap + c] : 0u;
    const uint4* p = reinterpret_cast<const uint4*>(Xh + (size_t)row * dpad) + l8;
    float lo = 0.f, hi = 0.f;
    for (int i = 0; i < dpad / 64; ++i) {
        const uint4 v = p[i * 8];
        const float* qv = rf_q + i * 64 + l8 * 8;
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {   // element 2e in the low half of the word, 2e + 1 in the high half
            refine_acc(__uint_as_float(w[e] << 16), qv[2 * e], lo, hi);
            refine_acc(__uint_as_float(w[e] & 0xFFFF0000u), qv[2 * e + 1], lo, hi);
        }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
        lo = __fadd_rd(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = __fadd_ru(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if (l8 == 0 && c < cap) {
        if (valid) {
            const float r = xres[row];
            const float a = fmaxf(__fsub_rd(__fsqrt_rd(lo), r), 0.f), b = __fadd_ru(__fsqrt_ru(hi), r);
            lo_out[(size_t)j * cap + c] = __fmul_rd(a, a);
            u_keys[(size_t)j * cap + c] = make_key_asc(__fmul_ru(b, b), (uint32_t)c);
        } else {
            u_keys[(size_t)j * cap + c] = KEY_PAD;
        }
    }
}

// Fetch rule.  u_top[j * P + P - 1] is U_(P), the P-th smallest U of query j (KEY_PAD: fewer than P candidates, fetch all).
// K1 rounds a distance D to D1 with |D1 - D| <= gamma D + eta (see fetch_rule_constants).  The P candidates of smallest U
// have D1 <= (1 + gamma) U_(P) + eta; a candidate with L > T = ((1 + gamma) U_(P) + 2 eta) / (1 - gamma) has
// D1 >= (1 - gamma) L - eta > (1 + gamma) U_(P) + eta: strictly worse, after K1's own rounding, than P fetched rows, so it
// cannot be in the top P whatever its ordinal.  Every candidate with L <= T is fetched (those P included: L <= U <= U_(P)).
__global__ void __launch_bounds__(256)
fetch_compact_kernel(const uint32_t* __restrict__ cand_count, const uint32_t* __restrict__ cand_rows, int cap,
                     const float* __restrict__ lo, const uint64_t* __restrict__ u_top, int P, float scale, float eta2,
                     uint32_t* __restrict__ fetch_count, uint32_t* __restrict__ fetch_rows)
{
    const int j = blockIdx.y, c = blockIdx.x * 256 + threadIdx.x;
    const int cnt = (int)min(cand_count[j], (uint32_t)cap);
    if (c >= cnt) return;
    const uint64_t kP = u_top[(size_t)j * P + (P - 1)];
    const float T = kP == KEY_PAD ? CUDART_INF_F : __fadd_ru(__fmul_ru(key_value_asc(kP), scale), eta2);
    if (lo[(size_t)j * cap + c] <= T) {
        const uint32_t pos = atomicAdd(&fetch_count[j], 1u);
        fetch_rows[(size_t)j * cap + pos] = cand_rows[(size_t)j * cap + c];
    }
}

// ------------------------------------------------------------------------ certificate
__global__ void certify_kernel(const float* __restrict__ Q, int dpad, int nq, int P, const float* __restrict__ thr,
                               const uint32_t* __restrict__ cand_count, int cap, const uint64_t* __restrict__ keys_out,
                               const uint32_t* __restrict__ xn_max_bits, float eps_rel, float slack_rel, int32_t* __restrict__ flags)
{
    const int j = blockIdx.x * blockDim.x / 32 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (j >= nq) return;
    float qn = 0.f;
    for (int i = lane; i < dpad; i += 32) { float v = Q[(size_t)j * dpad + i]; qn = fmaf(v, v, qn); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) qn += __shfl_xor_sync(0xffffffffu, qn, o);
    if (lane == 0) {
        const uint64_t kP = keys_out[(size_t)j * P + (P - 1)];
        const float xmax = __uint_as_float(*xn_max_bits);
        bool ok = cand_count[j] <= (uint32_t)cap && kP != KEY_PAD;
        if (ok) {
            const float dP = key_value_asc(kP);
            // |main-pass dot - exact dot| <= eps_rel |x| |q|, eps_rel = operand error + 2^-12 for the fp32 accumulation:
            //   TF32 (both operands truncated, 2^-10 each): 2^-9 + 2^-12
            //   bf16 (both operands rounded to nearest, 2^-8 each): 2^-7 + 2^-12
            // a pruned row has main-pass a >= thr, so its exact a >= thr - 2 eps; the sample pass only picks thr
            const float eps = eps_rel * sqrtf(xmax) * sqrtf(qn);
            const float slack = slack_rel * (1.f + qn + xmax);   // fp32 rounding elsewhere (certify_slack_rel)
            ok = dP <= thr[j] + qn - 2.f * eps - slack;
        }
        flags[j] = ok ? 1 : 0;
    }
}

// ------------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode()
{
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}
// 2-D map over [rows, dpad] fp32 (box 32 x box_rows) or bf16 (box 64 x box_rows) rows, 128B swizzle
static bool make_map(CUtensorMap* tm, const void* base, int64_t rows, int dpad, int box_rows, bool bf16 = false)
{
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t gdim[2] = {(cuuint64_t)dpad, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)dpad * (bf16 ? 2 : 4)};
    cuuint32_t box[2] = {(cuuint32_t)(bf16 ? 2 * TC_KBLOCK : TC_KBLOCK), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(tm, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// 3-D map over 128-byte pieces of 64 halves: piece p of row r at base + r * row_bytes + 128 p; box = one piece of
// box_rows rows (the pass's tile), 128B swizzle (the shared-memory image of a bf16 box of make_map).  bf16 rows: dpad / 64
// pieces of 2 dpad bytes; split rows: split_pieces(dpad) pieces of 4 dpad bytes.
// Split rows promote L2 fills to 128 B only: a 256-byte promotion would fetch the low halves beside every high-half piece.
static bool make_map_pieces(CUtensorMap* tm, const void* base, int64_t rows, int dpad, bool split, int box_rows)
{
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t gdim[3] = {(cuuint64_t)SPLIT_BLOCK, (cuuint64_t)(split ? split_pieces(dpad) : dpad / 64), (cuuint64_t)rows};
    cuuint64_t gstride[2] = {128, (cuuint64_t)dpad * (split ? 4 : 2)};
    cuuint32_t box[3] = {(cuuint32_t)SPLIT_BLOCK, 1, (cuuint32_t)box_rows};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     split ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

constexpr int64_t TC_MIN_ROWS = 262144;   // below this the exact scan is cheaper than sample + prune + rescore

bool dense_tc_supported(const DeviceInfo& di, int dpad)
{
    const size_t smem = TcCfg<256, TC_TF32S>::SMEM > Tc16Cfg<256>::SMEM ? TcCfg<256, TC_TF32S>::SMEM : Tc16Cfg<256>::SMEM;
    return di.cc_major == 9 && dpad % TC_KBLOCK == 0 && di.smem_optin >= smem && get_encode() != nullptr;
}

static int tc_target(int P, bool bf16 = false)
{
    int c = (bf16 ? 6 : 4) * P, lo = bf16 ? 1024 : 512;   // bf16 pruning needs a wider margin for its certificate
    return c < lo ? lo : (c > 3072 ? 3072 : c);
}
// Gamma(m)-distributed sample estimate (m = C/64 >= 8): 4x the target is a < 1e-8 overflow tail
static int tc_cap(int P) { return 4 * tc_target(P, true); }   // sized for either mode

struct TcWorkspace {   // carved out of the caller's byte buffer
    float* thr; uint32_t* cand_count; int32_t* flags; uint32_t* cand_rows; uint64_t* exact_keys; float* dump; uint16_t* q_bf16;
    float* lo; uint32_t* fetch_count; uint32_t* fetch_rows;   // host-resident rows only: refine bounds and fetch lists
};
static size_t tc_carve(TcWorkspace* w, unsigned char* base, int cap, int64_t S, bool host_rows = false)
{
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = (o + bytes + 255) & ~(size_t)255; return base ? base + at : nullptr; };
    unsigned char* p;
    p = take(256 * 4); if (w) w->thr = (float*)p;
    p = take(256 * 4); if (w) w->cand_count = (uint32_t*)p;
    p = take(256 * 4); if (w) w->flags = (int32_t*)p;
    p = take((size_t)256 * cap * 4); if (w) w->cand_rows = (uint32_t*)p;
    p = take((size_t)256 * cap * 8); if (w) w->exact_keys = (uint64_t*)p;
    p = take((size_t)256 * S * 4); if (w) w->dump = (float*)p;
    p = take((size_t)256 * 16384 * 2); if (w) w->q_bf16 = (uint16_t*)p;   // queries as bf16 (dim <= 16384)
    if (host_rows) {
        p = take((size_t)256 * cap * 4); if (w) w->lo = (float*)p;
        p = take(256 * 4); if (w) w->fetch_count = (uint32_t*)p;
        p = take((size_t)256 * cap * 4); if (w) w->fetch_rows = (uint32_t*)p;
    }
    return o;
}
static int64_t tc_sample_tiles(int64_t n_rows)
{
    int64_t n_tiles = (n_rows + TC_TILE_M - 1) / TC_TILE_M;
    return (n_tiles + TC_SAMPLE_STRIDE - 1) / TC_SAMPLE_STRIDE;
}
size_t dense_tc_workspace_bytes(const DeviceInfo&, int64_t n_rows, int P, bool host_rows)
{
    return tc_carve(nullptr, nullptr, tc_cap(P), tc_sample_tiles(n_rows) * TC_TILE_M, host_rows);
}
bool dense_tc_wants(int64_t n_rows, int batch) { return n_rows >= TC_MIN_ROWS && batch >= 16; }

// Constants of the fetch rule (fetch_compact_kernel).  K1 (dense_scan_kernel, rescore_kernel) computes D = sum (x_i - q_i)^2
// over nonnegative terms; every term passes through at most m = dpad / 32 + 7 roundings to nearest: its difference (squared:
// 2), its lane's FFMA chain (dpad / 32 steps), (p0 + p1) + (p2 + p3) (2) and the butterfly over lanes 4, 2, 1 (3).  With
// u = 2^-24 this gives |D1 - D| <= gamma D + eta, gamma = m u / (1 - m u) (Higham, Lemma 3.1); eta bounds what subnormal
// results add, at most 2^-150 each over at most dpad + 64 roundings (doubled to cover their propagation through later
// roundings).  scale >= (1 + gamma) / (1 - gamma) and eta2 >= 2 eta / (1 - gamma), both rounded up.
static void fetch_rule_constants(int dpad, float* scale, float* eta2)
{
    const double u = ldexp(1.0, -24), m = dpad / KRAG_LANES + 7;
    const double gamma = m * u / (1.0 - m * u);
    const double eta = (dpad + 64) * ldexp(1.0, -149);
    *scale = nextafterf((float)((1.0 + gamma) / (1.0 - gamma)), INFINITY);
    *eta2 = nextafterf((float)(2.0 * eta / (1.0 - gamma)), INFINITY);
}

// Slack of the certificate (certify_kernel): what fp32 rounding outside the main pass's dot product can move a pruned row's
// distance by, as a multiple of (1 + |q|^2 + |x|^2max).  A term passes through at most
//   mx = dpad / 128 + 9 roundings in |x|^2 (row_norms_kernel: its square and the 3 adds of its float4, the lane's dpad / 128
//        float4 adds, the 5-step butterfly),
//   mq = dpad / 32 + 5 in |q|^2 (certify_kernel: the lane's FFMA chain of dpad / 32 steps, the butterfly),
//   mk = dpad / 32 + 7 in K1's distance of the pruned row (fetch_rule_constants), whose D <= 2 (|x|^2 + |q|^2),
// and the epilogue's add (|2 acc + thr| <= 3 (|x|^2max + |q|^2)) and the certificate's three adds (operands below
// 2 (|x|^2max + |q|^2)) round 9 more times.  With u = 2^-24 that is (max(mx, mq) + 2 mk + 9) gamma-factors of u, rounded up;
// never below 4e-6, the constant it replaces, which rows from dpad 448 on outgrow (6.0e-6 at 768, 9.3e-5 at 16384).
static float certify_slack_rel(int dpad)
{
    const double u = ldexp(1.0, -24);
    const double mx = dpad / 128 + 9, mq = dpad / KRAG_LANES + 5, mk = dpad / KRAG_LANES + 7;
    const double m = (mx > mq ? mx : mq) + 2.0 * mk + 9.0;
    const double c = m * u / (1.0 - m * u);
    return c > 4e-6 ? nextafterf((float)c, INFINITY) : 4e-6f;
}

static std::atomic<int64_t> g_host_rows_fetched{0};
int64_t host_rows_fetched() { return g_host_rows_fetched.load(); }

// What a prune operand fixes besides its main kernel and rows (tc_pass): the kernel id krag_last_dense_kernel reports,
// whether the main pass multiplies bf16 operands (2 bytes per element, the bf16 error bound, a wider candidate margin) and
// the rows per tile of its kernel
struct TcOpInfo { int kernel_id; bool bf16; int tile_rows; };
static constexpr TcOpInfo TC_OPS[] = {{3, false, TC_TILE_M} /* TF32 */, {3, false, TC_TILE_M} /* TF32S */,
                                      {5, true, TC16_TILE_M} /* BF16_SPLIT */, {4, true, TC16_TILE_M} /* BF16_SHADOW */,
                                      {6, true, TC16_TILE_M} /* BF16_HOST */};

TcOp tc_operand(const DenseRows& r, bool shadow, bool tf32)
{
    if (r.host()) return TC_OP_BF16_HOST;
    if (shadow && r.bf16() && r.dpad % (2 * TC_KBLOCK) == 0) return TC_OP_BF16_SHADOW;   // bf16 k-blocks are 64 elements wide
    if (!r.split()) return TC_OP_TF32;
    return tf32 ? TC_OP_TF32S : TC_OP_BF16_SPLIT;
}

bool dense_tc_serves(const DeviceInfo& di, const DenseRows& r, TcOp op)
{
    return dense_tc_supported(di, r.dpad) && r.n >= TC_MIN_ROWS && r.n < (1ll << 31) &&
           (!TC_OPS[op].bf16 || r.dpad % (2 * TC_KBLOCK) == 0);   // bf16 k-blocks are 64 elements wide
}

// the TF32 kernels' map of device rows: 3-D pieces of split rows, 2-D fp32 rows otherwise
static bool make_rows_map(CUtensorMap* tm, const DenseRows& r)
{
    return r.split() ? make_map_pieces(tm, r.dev(), r.n, r.dpad, true, TC_TILE_M) : make_map(tm, r.dev(), r.n, r.dpad, TC_TILE_M);
}

// the queries as op's bf16 operand: rounded to nearest even, in the split rows' lane order inside each 64-element block for
// their high halves.  The TF32 kernels read the fp32 queries.
static void tc_queries(TcOp op, const float* q, int nq, int dpad, uint16_t* qh, cudaStream_t st)
{
    if (op == TC_OP_BF16_SPLIT) launch_bf16_split_order(q, qh, (int64_t)nq * dpad, st);
    else if (TC_OPS[op].bf16) launch_f32_to_bf16(q, qh, (int64_t)nq * dpad, st);
}

// op's prune kernel over n_tiles tiles, row_step rows apart: the main pass (rows below thr go to the candidate lists), or with
// DUMP the dump of a (dump_min: per 16-row group, the sample pass; otherwise per row, in the columns up to S).  The bf16
// kernel reads the high halves of split rows (its k-blocks step 2 pieces: high- and low-half pieces interleave) or bf16 rows,
// with the bf16 queries qh; the TF32 kernels read the maps tmX and tmQ.
template <int NQ, bool DUMP>
static void tc_prune(const DeviceInfo& di, const DenseRows& r, TcOp op, const CUtensorMap& tmX, const CUtensorMap& tmQ,
                     const uint16_t* qh, int nq, int64_t n_tiles, int row_step, const uint32_t* alive, const float* thr,
                     uint32_t* cand_count, uint32_t* cand_rows, int cap, float* dump, int64_t S, int dump_min, cudaStream_t st)
{
    using C16 = Tc16Cfg<NQ>;
    using C32 = TcCfg<NQ, TC_TF32>;
    using C32S = TcCfg<NQ, TC_TF32S>;
    static bool attr_set = false;
    if (!attr_set) {
        KRAG_CUDA(cudaFuncSetAttribute(dense_tc_bf16_kernel<NQ, DUMP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C16::SMEM));
        KRAG_CUDA(cudaFuncSetAttribute(dense_tc_kernel<NQ, TC_TF32, DUMP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C32::SMEM));
        KRAG_CUDA(cudaFuncSetAttribute(dense_tc_kernel<NQ, TC_TF32S, DUMP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C32S::SMEM));
        attr_set = true;
    }
    const int grid = (int)(n_tiles < di.sm_count ? n_tiles : di.sm_count);
    if (TC_OPS[op].bf16) {
        const bool split = op == TC_OP_BF16_SPLIT;
        CUtensorMap tmR, tmQh;
        if (!make_map(&tmQh, qh, nq, r.dpad, NQ, true) ||
            !make_map_pieces(&tmR, split ? (const void*)r.dev() : (const void*)r.bf16(), r.n, r.dpad, split, TC16_TILE_M))
            throw CudaError{cudaErrorUnknown, "cuTensorMapEncodeTiled(bf16 pass)", __FILE__, __LINE__};
        dense_tc_bf16_kernel<NQ, DUMP><<<grid, TC16_THREADS, C16::SMEM, st>>>(tmR, tmQh, r.n, r.dpad / C16::ELEMS, split ? 2 : 1, n_tiles,
                                                                              row_step, r.norms(), alive, thr, cand_count, cand_rows,
                                                                              cap, dump, S, dump_min);
    } else if (op == TC_OP_TF32S) {
        dense_tc_kernel<NQ, TC_TF32S, DUMP><<<grid, TC_THREADS, C32S::SMEM, st>>>(tmX, tmQ, r.n, r.dpad / C32S::ELEMS, n_tiles,
                                                                                  row_step / TC_TILE_M, r.norms(), alive, thr,
                                                                                  cand_count, cand_rows, cap, dump, S, dump_min);
    } else {
        dense_tc_kernel<NQ, TC_TF32, DUMP><<<grid, TC_THREADS, C32::SMEM, st>>>(tmX, tmQ, r.n, r.dpad / C32::ELEMS, n_tiles,
                                                                                row_step / TC_TILE_M, r.norms(), alive, thr,
                                                                                cand_count, cand_rows, cap, dump, S, dump_min);
    }
}

// One K2 pass of nq <= NQ queries.  Besides the main kernel, op decides the sample kernel (TC_TF32 on plain rows, TC_TF32S
// on split rows, the bf16 kernel on host rows' copy), the rescoring (from device rows, or refined on the copy and fetched
// from host rows) and eps_rel.
template <int NQ>
static void tc_pass(const DeviceInfo& di, const DenseRows& r, TcOp op, const CUtensorMap& tmX, const CUtensorMap& tmQ,
                    const uint32_t* alive, const float* q, int nq, int P, OrdMap ord_base, const TcWorkspace& w, int cap,
                    uint64_t* keys_out, cudaStream_t st)
{
    const int64_t n_rows = r.n;
    const int dpad = r.dpad;
    const bool host = op == TC_OP_BF16_HOST, bf16 = TC_OPS[op].bf16;
    tc_queries(op, q, nq, dpad, w.q_bf16, st);
    // 1. sample pass, dump a = |x|^2 - 2 x.q: one tile at the start of every TC_SAMPLE_STRIDE 128-row tiles, so every pass
    // samples the same rows first; bf16 on host rows (192-row tiles), TF32 otherwise (128-row tiles).  The sample pass only
    // chooses thr: its operands do not enter soundness.
    // the dump holds one value per (16-row group of a sampled tile, query): S_min per query
    const TcOp sample_op = host ? op : (r.split() ? TC_OP_TF32S : TC_OP_TF32);
    const int sample_m = TC_OPS[sample_op].tile_rows;
    const int64_t s_tiles = tc_sample_tiles(n_rows);
    const int64_t S_min = s_tiles * (sample_m / TC_DUMP_GROUP);
    tc_prune<NQ, true>(di, r, sample_op, tmX, tmQ, w.q_bf16, nq, s_tiles, TC_SAMPLE_STRIDE * TC_TILE_M, alive, nullptr, nullptr,
                       nullptr, 0, w.dump, S_min, 1, st);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    // 2. threshold admitting ~C rows: the m-th smallest of the sample, m = C * sample_fraction
    int64_t sampled_rows = 0;
    for (int64_t t = 0; t < s_tiles; ++t) {
        int64_t r0 = t * TC_SAMPLE_STRIDE * TC_TILE_M;
        sampled_rows += (r0 + sample_m <= n_rows) ? sample_m : (n_rows > r0 ? n_rows - r0 : 0);
    }
    int m = (int)((double)tc_target(P, bf16) * (double)sampled_rows / (double)n_rows + 0.5);
    if (m < 4) m = 4;
    if (m > 1024) m = 1024;
    // m-th smallest of the S_min group minima per query (a few thousand values: one block per query, one launch)
    if (m > (int)S_min) m = (int)S_min;
    if (m <= 256) sample_threshold_kernel<1024><<<dim3(NQ, 1), ST_THREADS, 0, st>>>(w.dump, S_min, m, nq, w.thr, nullptr);
    else sample_threshold_kernel<2048><<<dim3(NQ, 1), ST_THREADS, 0, st>>>(w.dump, S_min, m, nq, w.thr, nullptr);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    KRAG_CUDA(cudaMemsetAsync(w.cand_count, 0, 256 * 4, st));
    // 3. main pass: stream the corpus once, prune on the tensor cores
    dense_timer_begin(st, TC_OPS[op].kernel_id, n_rows * (int64_t)dpad * (bf16 ? 2 : 4), 2 * (int64_t)NQ * n_rows * dpad);
    const int tile = TC_OPS[op].tile_rows;
    tc_prune<NQ, false>(di, r, op, tmX, tmQ, w.q_bf16, nq, (n_rows + tile - 1) / tile, tile, alive, w.thr, w.cand_count, w.cand_rows,
                        cap, nullptr, 0, 0, st);
    dense_timer_end(st);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    // 4. exact fp32 rescoring of the survivors + top-P
    static bool rs_attr_set = false;
    if (!rs_attr_set) {   // the query row sits in shared memory: up to 64 KB at dim 16384, past the default 48 KB limit
        KRAG_CUDA(cudaFuncSetAttribute(rescore_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 4));
        KRAG_CUDA(cudaFuncSetAttribute(rescore_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 4));
        rs_attr_set = true;
    }
    dim3 rg((unsigned)((cap + 31) / 32), (unsigned)nq);
    if (host) {
        // refine on the bf16 copy, U_(P) per query (merged into keys_out, overwritten below), compact the candidates that
        // may be in the top P, rescore only those from the host rows
        static bool rf_attr_set = false;
        if (!rf_attr_set) {
            KRAG_CUDA(cudaFuncSetAttribute(refine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 4));
            KRAG_CUDA(cudaFuncSetAttribute(rescore_mapped_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 4));
            rf_attr_set = true;
        }
        refine_kernel<<<rg, 256, (size_t)dpad * 4, st>>>(r.bf16(), r.res(), dpad, q, w.cand_count, w.cand_rows, cap, w.lo, w.exact_keys);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        launch_merge(w.exact_keys, 1, cap, nq, P, cap, cap, keys_out, st);
        float scale, eta2;
        fetch_rule_constants(dpad, &scale, &eta2);
        KRAG_CUDA(cudaMemsetAsync(w.fetch_count, 0, 256 * 4, st));
        fetch_compact_kernel<<<dim3((unsigned)((cap + 255) / 256), (unsigned)nq), 256, 0, st>>>(
            w.cand_count, w.cand_rows, cap, w.lo, keys_out, P, scale, eta2, w.fetch_count, w.fetch_rows);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        rescore_mapped_kernel<<<rg, 256, (size_t)dpad * 4, st>>>(r.host_d(), dpad, q, w.fetch_count, w.fetch_rows, cap, ord_base,
                                                                 w.exact_keys);
    } else {
        if (r.split()) rescore_kernel<true><<<rg, 256, (size_t)dpad * 4, st>>>(r.dev(), dpad, q, w.cand_count, w.cand_rows, cap, ord_base, w.exact_keys);
        else rescore_kernel<false><<<rg, 256, (size_t)dpad * 4, st>>>(r.dev(), dpad, q, w.cand_count, w.cand_rows, cap, ord_base, w.exact_keys);
    }
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    launch_merge(w.exact_keys, 1, cap, nq, P, cap, cap, keys_out, st);
    // 5. certificate: the error bound of the main pass's operands (the sample pass only chooses thr, whatever its value)
    const float eps_rel = bf16 ? (0.0078125f + 0.000244140625f) : (0.001953125f + 0.000244140625f);
    certify_kernel<<<(nq * 32 + 255) / 256, 256, 0, st>>>(q, dpad, nq, P, w.thr, w.cand_count, cap, keys_out, r.norm_max(), eps_rel,
                                                          certify_slack_rel(dpad), w.flags);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

static std::atomic<int64_t> g_tc_fallback_queries{0};   // searches run concurrently (reader lock)
int64_t dense_tc_fallback_queries() { return g_tc_fallback_queries.load(); }

bool launch_dense_tc(const DeviceInfo& di, const DenseRows& r, TcOp op, const uint32_t* alive, const float* q, int batch,
                     int P, OrdMap ord_base, void* workspace, size_t workspace_bytes, uint64_t* part, const ScanStaging* sg,
                     uint64_t* keys_out, cudaStream_t st)
{
    const int64_t n_rows = r.n;
    const int dpad = r.dpad;
    const bool host = op == TC_OP_BF16_HOST;
    const int cap = tc_cap(P);
    TcWorkspace w;
    if (tc_carve(&w, (unsigned char*)workspace, cap, tc_sample_tiles(n_rows) * TC_TILE_M, host) > workspace_bytes) return false;
    // the maps of the TF32 kernels, which do not run on host rows; tmX is encoded once per call
    CUtensorMap tmX{}, tmQ{};
    if (!host && !make_rows_map(&tmX, r)) return false;
    std::vector<int32_t> flags(256);
    std::vector<uint32_t> fetched(host ? 256 : 0);   // host rows: rows each query fetched from host memory
    for (int b0 = 0; b0 < batch; b0 += 256) {
        const int nq = batch - b0 < 256 ? batch - b0 : 256;
        const int NQ = nq <= 64 ? 64 : (nq <= 128 ? 128 : 256);
        const float* qb = q + (size_t)b0 * dpad;
        if (!host && !make_map(&tmQ, qb, nq, dpad, NQ)) return false;
        uint64_t* ko = keys_out + (size_t)b0 * P;
        (NQ == 64 ? tc_pass<64> : NQ == 128 ? tc_pass<128> : tc_pass<256>)(di, r, op, tmX, tmQ, alive, qb, nq, P, ord_base, w, cap, ko, st);
        KRAG_CUDA(cudaMemcpyAsync(flags.data(), w.flags, sizeof(int32_t) * (size_t)nq, cudaMemcpyDeviceToHost, st));
        if (host) KRAG_CUDA(cudaMemcpyAsync(fetched.data(), w.fetch_count, sizeof(uint32_t) * (size_t)nq, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
        int nf = 0;
        for (int j = 0; j < nq; ++j)
            if (!flags[(size_t)j]) flags[(size_t)nf++] = j;   // flags[0, nf) now lists the uncertified queries
        // uncertified queries (rare) are re-run on the exact scan -- still on the GPU: one by one on device rows, together
        // in one streamed scan of host rows
        if (!host) {
            for (int i = 0; i < nf; ++i) {
                ++g_tc_fallback_queries;
                launch_dense_scan(di, r, alive, qb + (size_t)flags[(size_t)i] * dpad, 1, P, ord_base, part, ko + (size_t)flags[(size_t)i] * P, st);
            }
            continue;
        }
        int64_t rows = 0;
        for (int j = 0; j < nq; ++j) rows += fetched[(size_t)j] < (uint32_t)cap ? fetched[(size_t)j] : (uint32_t)cap;
        g_host_rows_fetched += rows;
        if (nf > 0) {
            g_tc_fallback_queries += nf;
            for (int i = 0; i < nf; ++i)
                KRAG_CUDA(cudaMemcpyAsync(sg->q_sel + (size_t)i * dpad, qb + (size_t)flags[(size_t)i] * dpad, sizeof(float) * (size_t)dpad,
                                          cudaMemcpyDeviceToDevice, st));
            launch_dense_scan(di, r, alive, sg->q_sel, nf, P, ord_base, part, sg->k_sel, st, sg);
            for (int i = 0; i < nf; ++i)
                KRAG_CUDA(cudaMemcpyAsync(ko + (size_t)flags[(size_t)i] * P, sg->k_sel + (size_t)i * P, sizeof(uint64_t) * (size_t)P,
                                          cudaMemcpyDeviceToDevice, st));
        }
    }
    return true;
}

// the dump's columns: the rows rounded up to 128 for every pass (the bf16 passes' dump covers them with 192-row tiles)
size_t dense_tc_debug_carve(TcDebugWs* w, unsigned char* base, int64_t n_rows, int dpad, int nq, int cap, int64_t* S_out,
                            int* nq_pad_out)
{
    const int NQ = nq <= 64 ? 64 : (nq <= 128 ? 128 : 256);
    const int64_t S = (n_rows + TC_TILE_M - 1) / TC_TILE_M * TC_TILE_M;
    *S_out = S;
    *nq_pad_out = NQ;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = (o + bytes + 255) & ~(size_t)255; return base ? base + at : nullptr; };
    TcDebugWs t{};
    t.q_bf16 = (uint16_t*)take((size_t)NQ * dpad * 2);
    if (cap == 0) {
        t.dump = (float*)take((size_t)NQ * S * 4);
    } else {
        t.thr = (float*)take((size_t)NQ * 4);
        t.cand_count = (uint32_t*)take((size_t)NQ * 4);
        t.cand_rows = (uint32_t*)take((size_t)NQ * cap * 4);
    }
    if (w) *w = t;
    return o;
}

bool dense_tc_debug_pass(const DeviceInfo& di, const DenseRows& r, TcOp op, const uint32_t* alive, const float* q, int nq,
                         const TcDebugWs& w, int cap, cudaStream_t st)
{
    if (!dense_tc_supported(di, r.dpad) || nq < 1 || nq > 256 || r.n < 1 || r.n >= (1ll << 31)) return false;
    if (op == TC_OP_BF16_SPLIT ? !r.split() : TC_OPS[op].bf16 && (!r.bf16() || r.dpad % (2 * TC_KBLOCK) != 0)) return false;
    const int NQ = nq <= 64 ? 64 : (nq <= 128 ? 128 : 256);
    // TF32: fp32 queries straight from the caller's rows; bf16: the queries converted as tc_pass converts them
    CUtensorMap tmX{}, tmQ{};
    if (!TC_OPS[op].bf16 && (!make_rows_map(&tmX, r) || !make_map(&tmQ, q, nq, r.dpad, NQ))) return false;
    tc_queries(op, q, nq, r.dpad, w.q_bf16, st);
    // cap == 0: as a sample pass, but over every row and the padding columns up to S; cap > 0: the main pass of tc_pass.
    // w holds the dump or the candidate lists, and null for the other.
    const int tile = TC_OPS[op].tile_rows;
    const int64_t S = (r.n + TC_TILE_M - 1) / TC_TILE_M * TC_TILE_M;
    if (cap > 0) KRAG_CUDA(cudaMemsetAsync(w.cand_count, 0, (size_t)NQ * 4, st));
    const bool dump = cap == 0;
    (NQ == 64 ? (dump ? tc_prune<64, true> : tc_prune<64, false>) : NQ == 128 ? (dump ? tc_prune<128, true> : tc_prune<128, false>)
                                                                   : (dump ? tc_prune<256, true> : tc_prune<256, false>))(
        di, r, op, tmX, tmQ, w.q_bf16, nq, ((dump ? S : r.n) + tile - 1) / tile, tile, alive, w.thr, w.cand_count, w.cand_rows, cap,
        w.dump, dump ? S : 0, 0, st);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    return true;
}

}  // namespace krag
