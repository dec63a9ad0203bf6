// embed.cu -- K5: BERT-family (bge-small / bge-base / bge-large, all-MiniLM, e5, gte; MPNet with its relative-position attention
// bias: all-mpnet-base-v2) encoder forward on the GPU.
//
// Replaces the torch / sentence-transformers forward behind
// presets/ragengine/embedding/huggingface_local_embedding.py:34-53 (LlamaIndex HuggingFaceEmbedding ->
// BertModel, CLS pooling, L2 normalisation; reached from embedding/base.py:25-26 on /retrieve and from
// VectorStoreIndex.from_documents on /index, vector_store/base.py:155-166).
//
//   tokens (packed, variable length: no padding rows)  ->  word+position+type embeddings -> LayerNorm
//   L x [ QKV GEMM -> attention -> O GEMM (+bias +residual) -> LayerNorm -> FFN1 GEMM (+bias, erf-GELU)
//         -> FFN2 GEMM (+bias +residual) -> LayerNorm ]  ->  CLS row or token mean (krag_embedder_set_pooling)  ->  L2 normalise
// Late interaction (ColBERT, krag_late_rerank): every token row of the last layer -> hidden x dim projection -> L2 normalise,
// then maxsim_kernel scores (query, passage) pairs from the kept token vectors, of the call's passages or of a LateStore.
//
// The four GEMMs per layer (24 S d^2 of the 24 S d^2 + 4 S^2 d flops) run on fp16 wgmma over split operands (see
// gemm_f16s_kernel) with fp32 accumulation in registers, operands staged by TMA; bias / GELU / residual are fused into
// the register epilogue.  LayerNorm and softmax are fp32 CUDA-core code; the attention products run on mma.sync
// (attention is 4 S^2 d: 2% of the flops at S = 32 queries).
#include <cuda_fp16.h>
#include <math_constants.h>

#include <cmath>
#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <tuple>
#include <string>
#include <vector>

#include "engine.h"
#include "embed_config.h"
#include "tc_ptx.cuh"
#include "common.cuh"

namespace krag {

// ------------------------------------------------------------------ GEMM: C = A . B^T (+bias)(gelu)(+res)
// A [M, K] (activations), B [N, K] (nn.Linear weight), C [M, N], row-major.  The tensor cores see fp16 operands, the result
// is fp32-accurate: every fp32 value v is carried as TWO fp16 numbers
//     hi = fp16(v),   lo = fp16((v - hi) * 2^11)          v = hi + lo * 2^-11  to ~2^-22 relative
// ("split" operands: producers write them next to / instead of the fp32 tensor, weights are split once at load time), and
//     A . B^T  =  hi_A . hi_B^T  +  2^-11 (hi_A . lo_B^T + lo_A . hi_B^T)          (lo . lo term: 2^-22, dropped)
// is three fp16 wgmma per K = 16 step into two register accumulators (main term / correction terms, combined in the
// epilogue; the scaling keeps the lo parts out of the fp16 subnormal range and the small terms out of the big
// accumulator's rounding).  fp16 products are exact in fp32, so what is left is the accumulation order -- the same kind of
// error an fp32 SIMT GEMM has.  Operand bytes per element are those of fp32 (2 + 2), the tensor work is 1.5x a TF32 GEMM's,
// and the result meets the reference's fp32 arithmetic (TF32 carried 10 mantissa bits: ~5e-3 on the unit-norm embedding).
//
// One kernel, gemm_f16s_kernel<BN>: 128 x BN output tiles (two consumer warpgroups of wgmma M = 64 rows), K cut into
// `splits` slices.  Work items (n fastest, so neighbouring CTAs share the A tile in L2, then m, then the K slice) are
// walked persistently by min(items, SMs) CTAs.  One TMA thread fills a ring of stages = one k-block of 64 halfs of hi_A,
// lo_A (128 rows each) and hi_B, lo_B (BN rows each).  splits == 1: bias / GELU / residual epilogue straight to the
// outputs; splits > 1: fp32 partials (main + 2^-11 correction) to ws[split][M][N], summed in split order by
// splitk_reduce_kernel (deterministic), which also applies bias / residual / LayerNorm and writes the split planes.
constexpr int GM_TILE = 128;
constexpr int GH_KB = 64;                   // halfs per k-block (128-byte swizzle row)
constexpr int GM_SLAB = GM_TILE * 128;      // 16 KB: 128 rows x 128 B
constexpr int GM_THREADS = 384;             // warpgroup 0: TMA producer, warpgroups 1-2: wgmma + epilogue
constexpr int GM_MAX_STAGES = 16;
constexpr int GM_SMEM_BUDGET = 200 * 1024;  // operand ring
constexpr float GH_LO_SCALE = 2048.f, GH_LO_INV = 1.f / 2048.f;

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

// ---- split fp16 operands
__device__ __forceinline__ uint16_t f2h_sat(float v)      // round to nearest even, finite saturation
{
    uint16_t h;
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(v));
    return h;
}
__device__ __forceinline__ float h2f(uint16_t h)
{
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
    return f;
}
__device__ __forceinline__ void split_f16(float v, uint16_t& hi, uint16_t& lo)
{
    hi = f2h_sat(v);
    lo = f2h_sat((v - h2f(hi)) * GH_LO_SCALE);
}
// 8 consecutive elements -> one 16-byte store into each plane
__device__ __forceinline__ void split_store8(const float* o, uint16_t* p_hi, uint16_t* p_lo)
{
    uint32_t a[4], b[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        uint16_t h0, l0, h1, l1;
        split_f16(o[2 * t], h0, l0); split_f16(o[2 * t + 1], h1, l1);
        a[t] = (uint32_t)h0 | ((uint32_t)h1 << 16); b[t] = (uint32_t)l0 | ((uint32_t)l1 << 16);
    }
    *reinterpret_cast<uint4*>(p_hi) = make_uint4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<uint4*>(p_lo) = make_uint4(b[0], b[1], b[2], b[3]);
}
// the hi plane alone: the fp16 operand of the single-plane (KRAG_PRECISION_FP16) products
__device__ __forceinline__ uint32_t hi_pack2(float a, float b) { return (uint32_t)f2h_sat(a) | ((uint32_t)f2h_sat(b) << 16); }
__device__ __forceinline__ void hi_store8(const float* o, uint16_t* p_hi)
{
    *reinterpret_cast<uint4*>(p_hi) = make_uint4(hi_pack2(o[0], o[1]), hi_pack2(o[2], o[3]), hi_pack2(o[4], o[5]), hi_pack2(o[6], o[7]));
}
__global__ void __launch_bounds__(256)
split_f16_kernel(const float* __restrict__ in, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, int64_t n8)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
        float o[8];
        const float4 x = reinterpret_cast<const float4*>(in)[2 * i], y = reinterpret_cast<const float4*>(in)[2 * i + 1];
        o[0] = x.x; o[1] = x.y; o[2] = x.z; o[3] = x.w; o[4] = y.x; o[5] = y.y; o[6] = y.z; o[7] = y.w;
        split_store8(o, hi + 8 * i, lo + 8 * i);
    }
}
void launch_split_f16(const float* in, uint16_t* hi, uint16_t* lo, int64_t n, cudaStream_t st)   // n % 8 == 0
{
    const int64_t n8 = n / 8;
    const int64_t want = (n8 + 255) / 256;
    split_f16_kernel<<<(unsigned)(want < 132 * 16 ? (want > 0 ? want : 1) : 132 * 16), 256, 0, st>>>(in, hi, lo, n8);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// what a GEMM epilogue writes: fp32 C and / or the split planes of C (operand of the next GEMM)
struct GemmOut {
    float* c;            // [M, N] fp32 or null
    uint16_t* hi;        // [M, N] split planes or null
    uint16_t* lo;        // PLANES == 1: not written
};

__device__ __forceinline__ float silu(float g) { return g / (1.f + expf(-g)); }
// EP_ROPE: (o0, o1) = elements i and i + dh/2 of a query or key head (the weight rows were permuted at finalize so that
// they are adjacent columns), rotated by the angle of (row position, pair i): q * cos + rotate_half(q) * sin in fp32
__device__ __forceinline__ void rope_rotate(float& o0, float& o1, float2 cs)
{
    const float a = o0 * cs.x - o1 * cs.y, b = o1 * cs.x + o0 * cs.y;
    o0 = a; o1 = b;
}

// PLANES == 2: the split product above.  PLANES == 1 (KRAG_PRECISION_FP16): the operands are the hi planes alone, fp16(v); a
// stage holds hi_A and hi_B (half the bytes: the ring is twice as deep), every K = 16 step is ONE wgmma into ONE
// accumulator (which leaves the registers for 128 x 256 tiles), and the epilogue writes fp32 C and / or the hi plane.
//
// EP (compile time) selects what the epilogue does after the bias (EpiArgs, engine.h):
//   EP_PLAIN   the BERT epilogue (+GELU) (+residual);
//   EP_ROPE    the QKV projection of a rotary encoder: columns below ep.rope_cols (Q and K) are rotated pairwise, a thread's
//              (c = 0, 1) pair being one (i, i + dh/2) pair of a head;
//   EP_SWIGLU  the gated FFN1: the weight rows are interleaved in blocks of 16 (8 up rows, then the 8 gate rows of the same
//              outputs), so column group j (even) holds up and group j + 1 the matching gate values; the epilogue writes
//              silu(gate) * up to [M][N / 2] outputs.
template <int BN, int PLANES, int EP = EP_PLAIN>
__global__ void __launch_bounds__(GM_THREADS, 1)
gemm_f16s_kernel(const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmA2,
                 const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmB2, int M, int N, int splits,
                 int kb_per_split, int n_stages, int b_evict_first, const float* __restrict__ bias, const float* residual,
                 int act_gelu, GemmOut out, float* __restrict__ ws, EpiArgs ep)
{
    constexpr int B_BYTES = BN * 128;                      // one plane of one weight k-block
    constexpr int STAGE_BYTES = PLANES * (GM_SLAB + B_BYTES);
    constexpr int R = BN / 2;                              // accumulators per thread and term
    constexpr int B_OFF = PLANES * GM_SLAB;                // hi_A (lo_A) hi_B (lo_B)
    extern __shared__ unsigned char gm_smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(gm_smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)n_stages * STAGE_BYTES);
    uint64_t* empty_bar = full_bar + GM_MAX_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m_tiles = (M + GM_TILE - 1) / GM_TILE, n_tiles = N / BN;
    const int total = m_tiles * n_tiles * splits;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA1); tma_prefetch_desc(&tmB1);
        if (PLANES == 2) { tma_prefetch_desc(&tmA2); tma_prefetch_desc(&tmB2); }
        for (int s = 0; s < n_stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
        fence_barrier_init();
    }
    pdl_launch_dependents();
    __syncthreads();
    pdl_wait();                        // everything above overlapped the previous kernel's tail

    if (warp < 4) {
        regs_dealloc<40>();
        if (threadIdx.x == 0) {
            const uint64_t pol_b = b_evict_first ? TMA_EVICT_FIRST : TMA_EVICT_LAST;
            int stage = 0; uint32_t phase = 0;
            for (int t = blockIdx.x; t < total; t += gridDim.x) {
                const int n0 = (t % n_tiles) * BN, m0 = ((t / n_tiles) % m_tiles) * GM_TILE;
                const int kb0 = (t / (n_tiles * m_tiles)) * kb_per_split;
                for (int i = 0; i < kb_per_split; ++i) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    unsigned char* s0 = smem + (size_t)stage * STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
                    const int k0 = (kb0 + i) * GH_KB;
                    tma_load_2d(s0, &tmA1, &full_bar[stage], k0, m0, TMA_EVICT_LAST);
                    if (PLANES == 2) tma_load_2d(s0 + GM_SLAB, &tmA2, &full_bar[stage], k0, m0, TMA_EVICT_LAST);
                    tma_load_2d(s0 + B_OFF, &tmB1, &full_bar[stage], k0, n0, pol_b);
                    if (PLANES == 2) tma_load_2d(s0 + B_OFF + B_BYTES, &tmB2, &full_bar[stage], k0, n0, pol_b);
                    if (++stage == n_stages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        regs_alloc<232>();
        const int wg = (warp >> 2) - 1, w = warp & 3;
        const int g = lane >> 2, q = lane & 3;
        const int r_lo = 64 * wg + 16 * w + g;             // this thread's accumulator rows: r_lo and r_lo + 8
        float acc_m[R], acc_c[PLANES == 2 ? R : 1];        // PLANES == 1: acc_c is never touched
        int stage = 0; uint32_t phase = 0;
        for (int t = blockIdx.x; t < total; t += gridDim.x) {
            const int n0 = (t % n_tiles) * BN, m0 = ((t / n_tiles) % m_tiles) * GM_TILE;
            const int split = t / (n_tiles * m_tiles);
            const bool rows_here = m0 + 64 * wg < M;        // a warpgroup whose 64 rows are all past M skips its MMAs
            for (int i = 0; i < kb_per_split; ++i) {
                mbar_wait(&full_bar[stage], phase);
                if (rows_here) {
                    const uint32_t s0 = smem_u32(smem + (size_t)stage * STAGE_BYTES);
                    const uint64_t a1 = wgmma_desc_sw128(s0 + wg * 64 * 128), a2 = wgmma_desc_sw128(s0 + GM_SLAB + wg * 64 * 128);
                    const uint64_t b1 = wgmma_desc_sw128(s0 + B_OFF), b2 = wgmma_desc_sw128(s0 + B_OFF + B_BYTES);
                    (void)a2; (void)b2;
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < GH_KB / 16; ++k) {   // K steps of 16 halfs = 32 bytes = 2 descriptor units
                        const uint32_t first = (uint32_t)((i | k) != 0);
                        wgmma_f16_ss<BN>(acc_m, a1 + 2 * k, b1 + 2 * k, first);
                        if constexpr (PLANES == 2) {
                            wgmma_f16_ss<BN>(acc_c, a1 + 2 * k, b2 + 2 * k, first);
                            wgmma_f16_ss<BN>(acc_c, a2 + 2 * k, b1 + 2 * k, 1u);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_operands<R>(acc_m);
                    if constexpr (PLANES == 2) wgmma_fence_operands<R>(acc_c);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[stage]);
                if (++stage == n_stages) { stage = 0; phase ^= 1; }
            }
            if (!rows_here) continue;
            // ===== epilogue straight from the registers: acc[4j + 2h + c] is (row r_lo + 8h, column n0 + 8j + 2q + c).
            // The bias and residual loads of EP_J column groups are issued together before any of them is used: one at a
            // time, each load's latency (the residual row comes from L2 or HBM) was paid in turn while the tensor cores idled.
            constexpr int EP_J = R / 4 < 8 ? R / 4 : 8;   // column groups per batch: all of a 128 x 32 tile's 4, else 8
            static_assert((R / 4) % EP_J == 0, "the batches cover the tile's column groups exactly");
            // element e of the tile's result: main + 2^-11 correction, or the one accumulator
            auto acc = [&](int e) {
                if constexpr (PLANES == 2) return fmaf(acc_c[e], GH_LO_INV, acc_m[e]);
                else return acc_m[e];
            };
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = m0 + r_lo + 8 * h;
                if (row >= M) continue;
                const size_t roff = (size_t)row * N;
                if (splits > 1) {
#pragma unroll
                    for (int j = 0; j < R / 4; ++j) {
                        const int col = n0 + 8 * j + 2 * q;
                        const float o0 = acc(4 * j + 2 * h), o1 = acc(4 * j + 2 * h + 1);
                        *reinterpret_cast<float2*>(ws + (size_t)split * M * N + roff + col) = make_float2(o0, o1);
                    }
                    continue;
                }
                // EP_SWIGLU writes rows of N / 2 outputs; EP_ROPE: this row's (cos, sin) pairs
                const size_t ooff = EP == EP_SWIGLU ? (size_t)row * (N / 2) : roff;
                const float2* rope_row = nullptr;
                if constexpr (EP == EP_ROPE) rope_row = reinterpret_cast<const float2*>(ep.rope) + (size_t)__ldg(ep.pos + row) * ep.half;
#pragma unroll
                for (int j0 = 0; j0 < R / 4; j0 += EP_J) {
                    float2 b2[EP_J], r2[EP_J], cs[EP == EP_ROPE ? EP_J : 1];
#pragma unroll
                    for (int u = 0; u < EP_J; ++u) {
                        const int col = n0 + 8 * (j0 + u) + 2 * q;
                        b2[u] = __ldg(reinterpret_cast<const float2*>(bias + col));
                        r2[u] = residual ? *reinterpret_cast<const float2*>(residual + roff + col) : make_float2(0.f, 0.f);
                        if constexpr (EP == EP_ROPE)
                            cs[u] = col < ep.rope_cols ? __ldg(rope_row + ((col & (2 * ep.half - 1)) >> 1)) : make_float2(1.f, 0.f);
                    }
#pragma unroll
                    for (int u = 0; u < EP_J; ++u) {
                        const int j = j0 + u;
                        int col = n0 + 8 * j + 2 * q;
                        float o0 = acc(4 * j + 2 * h), o1 = acc(4 * j + 2 * h + 1);
                        o0 += b2[u].x; o1 += b2[u].y;
                        if constexpr (EP == EP_SWIGLU) {
                            if (u & 1) continue;                     // the gate group: consumed with its up group
                            const float g0 = acc(4 * j + 4 + 2 * h) + b2[u + 1].x, g1 = acc(4 * j + 4 + 2 * h + 1) + b2[u + 1].y;
                            o0 = silu(g0) * o0; o1 = silu(g1) * o1;
                            col = n0 / 2 + 4 * j + 2 * q;              // output column of the 16-column block's 8 outputs
                        }
                        if (act_gelu) { o0 = gelu_erf(o0); o1 = gelu_erf(o1); }
                        if constexpr (EP == EP_ROPE) rope_rotate(o0, o1, cs[u]);
                        if (residual) { o0 += r2[u].x; o1 += r2[u].y; }
                        if (out.c) *reinterpret_cast<float2*>(out.c + ooff + col) = make_float2(o0, o1);
                        if constexpr (PLANES == 2) {
                            if (out.hi) {
                                uint16_t h0, l0, h1, l1;
                                split_f16(o0, h0, l0); split_f16(o1, h1, l1);
                                *reinterpret_cast<uint32_t*>(out.hi + ooff + col) = (uint32_t)h0 | ((uint32_t)h1 << 16);
                                *reinterpret_cast<uint32_t*>(out.lo + ooff + col) = (uint32_t)l0 | ((uint32_t)l1 << 16);
                            }
                        } else {
                            if (out.hi) *reinterpret_cast<uint32_t*>(out.hi + ooff + col) = hi_pack2(o0, o1);
                        }
                    }
                }
            }
        }
    }
}

// --------------------------------------------------------------------------- fp32 row kernels
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// one warp per row: y = LayerNorm(x) * g + b   (two-pass variance like torch); a lane owns groups of 8 consecutive
// elements (d % 8 == 0, d <= 1024) that it reads ONCE into registers; the fp32 row and the split fp16 planes are written
// with 32- / 16-byte stores
constexpr int LN_MAX_GROUPS = 4;      // 8-element groups per lane: d <= 32 * 4 * 8 = 1024
__device__ __forceinline__ void warp_layernorm_row(const float* __restrict__ x, float* __restrict__ y, uint16_t* __restrict__ y_hi,
                                                   uint16_t* __restrict__ y_lo, const float* __restrict__ g,
                                                   const float* __restrict__ b, int d, float eps, int lane)
{
    const int groups = d >> 3;
    float v[LN_MAX_GROUPS][8];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < LN_MAX_GROUPS; ++k) {
        const int gi = lane + 32 * k;
        if (gi < groups) {
            const float4 a = *reinterpret_cast<const float4*>(x + gi * 8), c = *reinterpret_cast<const float4*>(x + gi * 8 + 4);
            v[k][0] = a.x; v[k][1] = a.y; v[k][2] = a.z; v[k][3] = a.w; v[k][4] = c.x; v[k][5] = c.y; v[k][6] = c.z; v[k][7] = c.w;
            s += ((a.x + a.y) + (a.z + a.w)) + ((c.x + c.y) + (c.z + c.w));
        }
    }
    const float mean = warp_sum(s) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < LN_MAX_GROUPS; ++k) {
        if (lane + 32 * k < groups) {
#pragma unroll
            for (int t = 0; t < 8; ++t) { v[k][t] -= mean; }
            q += ((v[k][0] * v[k][0] + v[k][1] * v[k][1]) + (v[k][2] * v[k][2] + v[k][3] * v[k][3])) +
                 ((v[k][4] * v[k][4] + v[k][5] * v[k][5]) + (v[k][6] * v[k][6] + v[k][7] * v[k][7]));
        }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
#pragma unroll
    for (int k = 0; k < LN_MAX_GROUPS; ++k) {
        const int gi = lane + 32 * k;
        if (gi < groups) {
            const float4 g0 = __ldg(reinterpret_cast<const float4*>(g + gi * 8)), g1 = __ldg(reinterpret_cast<const float4*>(g + gi * 8 + 4));
            const float4 b0 = __ldg(reinterpret_cast<const float4*>(b + gi * 8)), b1 = __ldg(reinterpret_cast<const float4*>(b + gi * 8 + 4));
            float o[8];
            o[0] = v[k][0] * rstd * g0.x + b0.x; o[1] = v[k][1] * rstd * g0.y + b0.y; o[2] = v[k][2] * rstd * g0.z + b0.z; o[3] = v[k][3] * rstd * g0.w + b0.w;
            o[4] = v[k][4] * rstd * g1.x + b1.x; o[5] = v[k][5] * rstd * g1.y + b1.y; o[6] = v[k][6] * rstd * g1.z + b1.z; o[7] = v[k][7] * rstd * g1.w + b1.w;
            if (y) {
                *reinterpret_cast<float4*>(y + gi * 8) = make_float4(o[0], o[1], o[2], o[3]);
                *reinterpret_cast<float4*>(y + gi * 8 + 4) = make_float4(o[4], o[5], o[6], o[7]);
            }
            if (y_lo) split_store8(o, y_hi + gi * 8, y_lo + gi * 8);
            else if (y_hi) hi_store8(o, y_hi + gi * 8);
        }
    }
}

__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, float* __restrict__ y, uint16_t* __restrict__ y_hi, uint16_t* __restrict__ y_lo,
                 const float* __restrict__ g, const float* __restrict__ b, int rows, int d, float eps)
{
    pdl_launch_dependents();
    pdl_wait();
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (r >= rows) return;
    warp_layernorm_row(x + (size_t)r * d, y ? y + (size_t)r * d : nullptr, y_hi ? y_hi + (size_t)r * d : nullptr,
                       y_lo ? y_lo + (size_t)r * d : nullptr, g, b, d, eps, lane);
}

// embeddings: x[t] = LN(word[id] + pos[p] + type[typ[t]]); one warp per token; scratch row in shared memory.  typ null (single
// sequences): type row 0 for every token; a cross-encoder pair has type 0 through its first [SEP] and type 1 after it.
// POS = false (rotary encoders): no position row, x[t] = LN(word[id] + type[typ[t]]); pos and pemb are not read.
template <bool POS>
__global__ void __launch_bounds__(256)
embed_ln_kernel(const int32_t* __restrict__ tok, const int32_t* __restrict__ pos, const int32_t* __restrict__ typ,
                const float* __restrict__ word, const float* __restrict__ pemb, const float* __restrict__ temb, const float* __restrict__ g,
                const float* __restrict__ b, float* __restrict__ x, uint16_t* __restrict__ x_hi, uint16_t* __restrict__ x_lo,
                int n_tok, int d, int vocab, float eps)
{
    extern __shared__ float e_sm[];   // [8][d]
    pdl_launch_dependents();
    pdl_wait();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * 8 + w;
    if (t >= n_tok) return;
    float* row = e_sm + (size_t)w * d;
    int id = tok[t];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const float* wr = word + (size_t)id * d;
    const float* pr = POS ? pemb + (size_t)pos[t] * d : nullptr;
    const float* tr = typ ? temb + (size_t)typ[t] * d : temb;
    if constexpr (POS) {
        for (int i = lane; i < d; i += 32) row[i] = (wr[i] + tr[i]) + pr[i];   // torch: inputs_embeds + token_type + position
    } else {
        for (int i = lane; i < d; i += 32) row[i] = wr[i] + tr[i];
    }
    __syncwarp();
    warp_layernorm_row(row, x + (size_t)t * d, x_hi + (size_t)t * d, x_lo ? x_lo + (size_t)t * d : nullptr, g, b, d, eps, lane);
}

// split-K epilogue: out[row] = f(sum_s ws[s][row] + bias) (+GELU) (+residual), optionally followed by LayerNorm over
// the row (N <= 1024).  One 256-thread block per row, one float4 column group per thread: the `splits` partial loads
// of a thread are independent (all in flight at once) -- with a few rows this kernel is pure load latency.
// `residual` and `out` may alias (a thread reads its residual elements before it writes them).
// EP as in gemm_f16s_kernel (no LayerNorm with EP_ROPE / EP_SWIGLU): EP_ROPE rotates the float4's two (i, i + dh/2) pairs
// below ep.rope_cols; EP_SWIGLU reads output group c's up columns and the gate columns 8 to their right and writes
// silu(gate) * up to rows of N / 2.
constexpr int SK_MAX_SPLITS = 8;
template <int EP = EP_PLAIN>
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ ws, int splits, int M, int N, const float* __restrict__ bias, const float* residual,
                     int act_gelu, const float* __restrict__ ln_g, const float* __restrict__ ln_b, float eps, float* out,
                     uint16_t* __restrict__ out_hi, uint16_t* __restrict__ out_lo, EpiArgs ep)
{
    __shared__ float s_red[2][8];
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const size_t plane = (size_t)M * N;
    const int ldo = EP == EP_SWIGLU ? N / 2 : N;              // output row stride
    const float* w0 = ws + (size_t)row * N;
    auto element = [&](int c) {
        float4 p[SK_MAX_SPLITS];
#pragma unroll
        for (int sp = 0; sp < SK_MAX_SPLITS; ++sp)
            if (sp < splits) p[sp] = *reinterpret_cast<const float4*>(w0 + (size_t)sp * plane + c);
        float4 s = p[0];
#pragma unroll
        for (int sp = 1; sp < SK_MAX_SPLITS; ++sp)
            if (sp < splits) { s.x += p[sp].x; s.y += p[sp].y; s.z += p[sp].z; s.w += p[sp].w; }
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + c));
        s.x += b4.x; s.y += b4.y; s.z += b4.z; s.w += b4.w;
        if (act_gelu) { s.x = gelu_erf(s.x); s.y = gelu_erf(s.y); s.z = gelu_erf(s.z); s.w = gelu_erf(s.w); }
        if (residual) {
            const float4 r = *reinterpret_cast<const float4*>(residual + (size_t)row * N + c);
            s.x += r.x; s.y += r.y; s.z += r.z; s.w += r.w;
        }
        return s;
    };
    auto store4 = [&](int c, const float4& o) {
        if (out) *reinterpret_cast<float4*>(out + (size_t)row * ldo + c) = o;
        if (out_hi && !out_lo) {
            *reinterpret_cast<uint2*>(out_hi + (size_t)row * ldo + c) = make_uint2(hi_pack2(o.x, o.y), hi_pack2(o.z, o.w));
        } else if (out_hi) {
            uint16_t h0, l0, h1, l1, h2, l2, h3, l3;
            split_f16(o.x, h0, l0); split_f16(o.y, h1, l1); split_f16(o.z, h2, l2); split_f16(o.w, h3, l3);
            *reinterpret_cast<uint2*>(out_hi + (size_t)row * ldo + c) = make_uint2((uint32_t)h0 | ((uint32_t)h1 << 16), (uint32_t)h2 | ((uint32_t)h3 << 16));
            *reinterpret_cast<uint2*>(out_lo + (size_t)row * ldo + c) = make_uint2((uint32_t)l0 | ((uint32_t)l1 << 16), (uint32_t)l2 | ((uint32_t)l3 << 16));
        }
    };
    if constexpr (EP == EP_SWIGLU) {
        for (int c = tid * 4; c < ldo; c += 1024) {
            const int cu = (c >> 3) * 16 + (c & 7);                // up columns of outputs c .. c + 3; the gate's are cu + 8
            const float4 u = element(cu), g = element(cu + 8);
            store4(c, make_float4(silu(g.x) * u.x, silu(g.y) * u.y, silu(g.z) * u.z, silu(g.w) * u.w));
        }
        return;
    } else if constexpr (EP == EP_ROPE) {
        const float2* rope_row = reinterpret_cast<const float2*>(ep.rope) + (size_t)__ldg(ep.pos + row) * ep.half;
        for (int c = tid * 4; c < N; c += 1024) {
            float4 o = element(c);
            if (c < ep.rope_cols) {
                const int i = (c & (2 * ep.half - 1)) >> 1;       // pairs (c, c + 1) and (c + 2, c + 3): i and i + 1
                rope_rotate(o.x, o.y, __ldg(rope_row + i));
                rope_rotate(o.z, o.w, __ldg(rope_row + i + 1));
            }
            store4(c, o);
        }
        return;
    }
    if (ln_g == nullptr) {
        for (int c = tid * 4; c < N; c += 1024) store4(c, element(c));
        return;
    }
    const int c = tid * 4;                         // N <= 1024: at most one column group per thread
    const bool on = c < N;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (on) v = element(c);
    float sum = warp_sum((v.x + v.y) + (v.z + v.w));
    if (lane == 0) s_red[0][warp] = sum;
    __syncthreads();
    sum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) sum += s_red[0][w];
    const float mean = sum / (float)N;
    const float a = v.x - mean, b = v.y - mean, cc = v.z - mean, dd = v.w - mean;
    float var = on ? (a * a + b * b) + (cc * cc + dd * dd) : 0.f;
    var = warp_sum(var);
    if (lane == 0) s_red[1][warp] = var;
    __syncthreads();
    var = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) var += s_red[1][w];
    const float rstd = rsqrtf(var / (float)N + eps);
    if (on) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(ln_g + c)), be = __ldg(reinterpret_cast<const float4*>(ln_b + c));
        float4 o;
        o.x = a * rstd * g.x + be.x; o.y = b * rstd * g.y + be.y; o.z = cc * rstd * g.z + be.z; o.w = dd * rstd * g.w + be.w;
        store4(c, o);
    }
}

// ------------------------------------------------------------------------------- attention
// ---- tensor-core attention: mma.sync m16n8k16 on the split fp16 planes the QKV projection writes, fp32 accumulators and
// fp32 max-subtracted softmax.  Every product is the error-compensated 3-MMA form of the GEMMs above:
//   A . B^T = hiA.hiB + 2^-11 (hiA.loB + loA.hiB).
// One CTA per (sequence, head, block of 16 x WARPS query rows), one warp per 16 rows (flash-style: online softmax over key
// blocks of KB keys; probabilities go from the score accumulators straight into the A fragments of P.V).  K and V planes
// of a key block are staged in shared memory by cp.async (STAGES = 2: the next block flies during the current one) and read
// with ldmatrix (V transposed on the fly), rows padded by 16 bytes so the 8 x 16-byte row reads hit 8 distinct bank groups.
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_f16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16_zfill(uint32_t smem_dst, const void* gsrc, bool valid)
{
    const int sz = valid ? 16 : 0;                        // 0 source bytes: the 16 destination bytes are zero-filled
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t& hi, uint32_t& lo)
{
    uint16_t h0, l0, h1, l1;
    split_f16(a, h0, l0); split_f16(b, h1, l1);
    hi = (uint32_t)h0 | ((uint32_t)h1 << 16); lo = (uint32_t)l0 | ((uint32_t)l1 << 16);
}
__device__ __forceinline__ void am_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void am_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// PLANES == 1 (KRAG_PRECISION_FP16): only the hi planes are staged and every product is one MMA on them; same key blocking,
// same fp32 softmax.
//
// REL (MPNet): every score gets its head's learned bias at the key - query distance, clamped to [-REL_MAX, REL_MAX]:
// rel_tab [heads][REL_TAB] holds it at index distance + REL_MAX (embedder_finalize builds it from the 32-bucket table).  The
// head's row is staged after the K / V stages in shared memory.  REL = false ignores rel_tab and is the BERT kernel.
//
// KVL (ColBERT queries with attend_to_mask_tokens false): sequence b's keys are its first kv_len[b] rows (1 <= kv_len[b] <=
// len); keys at or past it score -inf before the online softmax, key blocks past it are not visited, and every row of the
// sequence stays a query row.  KVL = false ignores kv_len.
constexpr int REL_MAX = 128, REL_TAB = 2 * REL_MAX + 1;
template <int DH, int WARPS, int KB, int STAGES, int PLANES> struct AmCfg {
    static constexpr int LDH = DH + 8;                                   // row stride in halfs (16 bytes of padding)
    static constexpr int Q_HALFS = PLANES * 16 * WARPS * LDH;            // hi | lo
    static constexpr int KV_HALFS = PLANES * KB * LDH;                   // hi | lo of one operand of one stage
    static constexpr size_t SMEM = 2 * (size_t)(Q_HALFS + 2 * STAGES * KV_HALFS);
};
template <int DH, int WARPS, int KB, int STAGES, int PLANES, bool REL, bool KVL>
__global__ void __launch_bounds__(WARPS * 32)
attention_mma_kernel(const uint16_t* __restrict__ qkv_hi, const uint16_t* __restrict__ qkv_lo, const int32_t* __restrict__ seq_off,
                     uint16_t* __restrict__ out_hi, uint16_t* __restrict__ out_lo, int d, int heads, const float* __restrict__ rel_tab,
                     const int32_t* __restrict__ kv_len)
{
    using Cfg = AmCfg<DH, WARPS, KB, STAGES, PLANES>;
    constexpr int LDH = Cfg::LDH, QROWS = 16 * WARPS, THREADS = WARPS * 32, CH = DH / 8 /* 16-byte chunks per row */;
    extern __shared__ __align__(16) uint16_t am_sm[];
    uint16_t* sQ = am_sm;                                  // [2][QROWS][LDH]
    uint16_t* sK = sQ + Cfg::Q_HALFS;                      // [STAGES][2][KB][LDH]
    uint16_t* sV = sK + STAGES * Cfg::KV_HALFS;            // [STAGES][2][KB][LDH]
    float* sRel = reinterpret_cast<float*>(sV + STAGES * Cfg::KV_HALFS);   // REL: [REL_TAB]
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.z, h = blockIdx.y;
    const int t0 = seq_off[b], len = seq_off[b + 1] - t0;
    const int r0 = blockIdx.x * QROWS;
    if (r0 >= len) return;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const size_t ld = (size_t)3 * d;
    // rows [row0, row0 + nrows) of one of Q | K | V (column offset `col`) of this head, both planes -> dst[2][nrows][LDH]
    auto stage_rows = [&](uint16_t* dst, int nrows, int row0, int col) {
        for (int i = tid; i < PLANES * nrows * CH; i += THREADS) {
            const int pl = i / (nrows * CH), rem = i % (nrows * CH), r = rem / CH, ch = rem % CH;
            const bool valid = row0 + r < len;
            const uint16_t* src = (pl ? qkv_lo : qkv_hi) + (valid ? (size_t)(t0 + row0 + r) * ld + col + h * DH + ch * 8 : 0);
            cp_async16_zfill(smem_u32(dst + ((size_t)pl * nrows + r) * LDH + ch * 8), src, valid);
        }
    };
    auto stage_kv = [&](int kb, int stage) {
        stage_rows(sK + stage * Cfg::KV_HALFS, KB, kb * KB, d);
        stage_rows(sV + stage * Cfg::KV_HALFS, KB, kb * KB, 2 * d);
        am_commit();
    };
    stage_rows(sQ, QROWS, r0, 0);
    stage_kv(0, 0);
    if constexpr (REL) {                                   // read after the first key block's __syncthreads
        for (int i = tid; i < REL_TAB; i += THREADS) sRel[i] = rel_tab[(size_t)h * REL_TAB + i];
    }
    const int n_keys = KVL ? kv_len[b] : len;
    const int nkb = (n_keys + KB - 1) / KB;
    uint32_t qh[DH / 16][4], ql[DH / 16][4];
    float om[DH / 8][4], oc[PLANES == 2 ? DH / 8 : 1][4];  // output accumulators: main and correction products
#pragma unroll
    for (int j = 0; j < DH / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            om[j][e] = 0.f;
            if constexpr (PLANES == 2) oc[j][e] = 0.f;
        }
    float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};     // rows g and g + 8 of the warp's 16
    const float scale = rsqrtf((float)DH);
    for (int kb = 0; kb < nkb; ++kb) {
        const int stage = STAGES == 2 ? (kb & 1) : 0;
        if (STAGES == 2 && kb + 1 < nkb) { stage_kv(kb + 1, (kb + 1) & 1); am_wait<1>(); } else am_wait<0>();
        __syncthreads();
        if (kb == 0) {
#pragma unroll
            for (int kk = 0; kk < DH / 16; ++kk) {
                const uint32_t a = smem_u32(sQ + (size_t)(warp * 16 + (lane & 15)) * LDH + kk * 16 + (lane >> 4) * 8);
                ldsm_x4(a, qh[kk][0], qh[kk][1], qh[kk][2], qh[kk][3]);
                if constexpr (PLANES == 2) ldsm_x4(a + 2 * QROWS * LDH, ql[kk][0], ql[kk][1], ql[kk][2], ql[kk][3]);
            }
        }
        const uint16_t* kH = sK + stage * Cfg::KV_HALFS;
        const uint16_t* vH = sV + stage * Cfg::KV_HALFS;
        // ---- scores: the two correction products first, scaled by 2^-11, then the main product on top (one accumulator)
        float s[KB / 8][4];
#pragma unroll
        for (int j = 0; j < KB / 8; ++j) {
            s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
            if constexpr (PLANES == 2) {
#pragma unroll
                for (int k2 = 0; k2 < DH / 32; ++k2) {
                    const uint32_t a = smem_u32(kH + (size_t)(j * 8 + (lane & 7)) * LDH + k2 * 32 + (lane >> 3) * 8);
                    uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
                    ldsm_x4(a, h0, h1, h2, h3);
                    ldsm_x4(a + 2 * KB * LDH, l0, l1, l2, l3);
                    mma_f16(s[j], qh[2 * k2], l0, l1); mma_f16(s[j], ql[2 * k2], h0, h1);
                    mma_f16(s[j], qh[2 * k2 + 1], l2, l3); mma_f16(s[j], ql[2 * k2 + 1], h2, h3);
                }
                s[j][0] *= GH_LO_INV; s[j][1] *= GH_LO_INV; s[j][2] *= GH_LO_INV; s[j][3] *= GH_LO_INV;
            }
#pragma unroll
            for (int k2 = 0; k2 < DH / 32; ++k2) {
                const uint32_t a = smem_u32(kH + (size_t)(j * 8 + (lane & 7)) * LDH + k2 * 32 + (lane >> 3) * 8);
                uint32_t h0, h1, h2, h3;
                ldsm_x4(a, h0, h1, h2, h3);
                mma_f16(s[j], qh[2 * k2], h0, h1); mma_f16(s[j], qh[2 * k2 + 1], h2, h3);
            }
        }
        // ---- online softmax (fp32): thread (g, t) holds columns 2t, 2t+1 of every 8-key tile for rows g (e = 0, 1) and g + 8 (e = 2, 3)
        const int k0 = kb * KB;
        const int dist0 = k0 + 2 * t - (r0 + warp * 16 + g);     // REL: key - query of element (j, e) is dist0 + 8j + (e & 1) - 8(e >> 1)
        float mx[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
        for (int j = 0; j < KB / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const bool in = k0 + j * 8 + 2 * t + (e & 1) < n_keys;
                if constexpr (REL) {                       // transformers' order: scale, then + position bias, then the mask
                    const int c = dist0 + j * 8 + (e & 1) - 8 * (e >> 1);
                    const float bias = sRel[min(max(c, -REL_MAX), REL_MAX) + REL_MAX];
                    s[j][e] = in ? fmaf(s[j][e], scale, bias) : -CUDART_INF_F;
                } else {
                    s[j][e] = in ? s[j][e] * scale : -CUDART_INF_F;
                }
                mx[e >> 1] = fmaxf(mx[e >> 1], s[j][e]);
            }
        float corr[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);            // finite: every key block holds at least one valid key
            corr[r] = expf(m_run[r] - m_new);                      // exp(-inf) = 0 on the first block
            m_run[r] = m_new;
        }
        float sum[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < KB / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float p = expf(s[j][e] - m_run[e >> 1]);     // masked columns: exp(-inf) = 0
                s[j][e] = p;
                sum[e >> 1] += p;
            }
        l_run[0] = l_run[0] * corr[0] + sum[0];                    // per-thread partial row sums (reduced over t at the end)
        l_run[1] = l_run[1] * corr[1] + sum[1];
#pragma unroll
        for (int j = 0; j < DH / 8; ++j) {
            om[j][0] *= corr[0]; om[j][1] *= corr[0]; om[j][2] *= corr[1]; om[j][3] *= corr[1];
            if constexpr (PLANES == 2) { oc[j][0] *= corr[0]; oc[j][1] *= corr[0]; oc[j][2] *= corr[1]; oc[j][3] *= corr[1]; }
        }
        // ---- out += P . V : the score accumulators of key tiles 2u, 2u+1 ARE the A fragment of 16-key step u
#pragma unroll
        for (int u = 0; u < KB / 16; ++u) {
            uint32_t ph[4], pl[4];
            if constexpr (PLANES == 2) {
                split_pack2(s[2 * u][0], s[2 * u][1], ph[0], pl[0]);
                split_pack2(s[2 * u][2], s[2 * u][3], ph[1], pl[1]);
                split_pack2(s[2 * u + 1][0], s[2 * u + 1][1], ph[2], pl[2]);
                split_pack2(s[2 * u + 1][2], s[2 * u + 1][3], ph[3], pl[3]);
            } else {
                ph[0] = hi_pack2(s[2 * u][0], s[2 * u][1]); ph[1] = hi_pack2(s[2 * u][2], s[2 * u][3]);
                ph[2] = hi_pack2(s[2 * u + 1][0], s[2 * u + 1][1]); ph[3] = hi_pack2(s[2 * u + 1][2], s[2 * u + 1][3]);
            }
#pragma unroll
            for (int jp = 0; jp < DH / 16; ++jp) {
                const uint32_t a = smem_u32(vH + (size_t)(u * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDH + jp * 16 + (lane >> 4) * 8);
                uint32_t h0, h1, h2, h3;
                ldsm_x4_trans(a, h0, h1, h2, h3);
                if constexpr (PLANES == 2) {
                    uint32_t l0, l1, l2, l3;
                    ldsm_x4_trans(a + 2 * KB * LDH, l0, l1, l2, l3);
                    mma_f16(om[2 * jp], ph, h0, h1); mma_f16(oc[2 * jp], ph, l0, l1); mma_f16(oc[2 * jp], pl, h0, h1);
                    mma_f16(om[2 * jp + 1], ph, h2, h3); mma_f16(oc[2 * jp + 1], ph, l2, l3); mma_f16(oc[2 * jp + 1], pl, h2, h3);
                } else {
                    mma_f16(om[2 * jp], ph, h0, h1);
                    mma_f16(om[2 * jp + 1], ph, h2, h3);
                }
            }
        }
        __syncthreads();                                           // the stage is free again
        if (STAGES == 1 && kb + 1 < nkb) stage_kv(kb + 1, 0);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float inv[2] = {1.f / l_run[0], 1.f / l_run[1]};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = r0 + warp * 16 + g + 8 * r;
        if (row >= len) continue;
        const size_t ob = (size_t)(t0 + row) * d + h * DH + 2 * t;
#pragma unroll
        for (int j = 0; j < DH / 8; ++j) {
            if constexpr (PLANES == 2) {
                uint32_t hi, lo;
                split_pack2(fmaf(oc[j][2 * r], GH_LO_INV, om[j][2 * r]) * inv[r], fmaf(oc[j][2 * r + 1], GH_LO_INV, om[j][2 * r + 1]) * inv[r], hi, lo);
                *reinterpret_cast<uint32_t*>(out_hi + ob + j * 8) = hi;
                *reinterpret_cast<uint32_t*>(out_lo + ob + j * 8) = lo;
            } else {
                *reinterpret_cast<uint32_t*>(out_hi + ob + j * 8) = hi_pack2(om[j][2 * r] * inv[r], om[j][2 * r + 1] * inv[r]);
            }
        }
    }
}

// the [CLS] rows of the residual stream x and of the attention context planes into row b of compact buffers: one warp per
// sequence, d % 128 == 0
__global__ void __launch_bounds__(256)
gather_cls_kernel(const float* __restrict__ x, const uint16_t* __restrict__ c_hi, const uint16_t* __restrict__ c_lo,
                  const int32_t* __restrict__ seq_off, float* __restrict__ gx, uint16_t* __restrict__ g_hi, uint16_t* __restrict__ g_lo,
                  int batch, int d)
{
    pdl_launch_dependents();
    pdl_wait();
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= batch) return;
    const size_t src = (size_t)seq_off[b] * d, dst = (size_t)b * d;
    for (int i = 4 * lane; i < d; i += 128) *reinterpret_cast<float4*>(gx + dst + i) = *reinterpret_cast<const float4*>(x + src + i);
    for (int i = 8 * lane; i < d; i += 256) {
        *reinterpret_cast<uint4*>(g_hi + dst + i) = *reinterpret_cast<const uint4*>(c_hi + src + i);
        if (g_lo) *reinterpret_cast<uint4*>(g_lo + dst + i) = *reinterpret_cast<const uint4*>(c_lo + src + i);
    }
}

// CLS pooling + L2 normalisation (F.normalize, eps 1e-12): one warp per sequence.  seq_off null: x holds the [CLS] rows
// only, row b for sequence b.
__global__ void __launch_bounds__(256)
cls_normalize_kernel(const float* __restrict__ x, const int32_t* __restrict__ seq_off, float* __restrict__ out, int batch, int d,
                     int ld_out)
{
    pdl_launch_dependents();
    pdl_wait();
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= batch) return;
    const float* row = x + (size_t)(seq_off ? seq_off[b] : b) * d;
    float s = 0.f;
    for (int i = lane; i < d; i += 32) s = fmaf(row[i], row[i], s);
    const float n = fmaxf(sqrtf(warp_sum(s)), 1e-12f);
    for (int i = lane; i < d; i += 32) out[(size_t)b * ld_out + i] = row[i] / n;
}

// mean pooling + L2 normalisation (sentence-transformers Pooling(pooling_mode_mean_tokens) over every token of the
// sequence, [CLS] and [SEP] included, then F.normalize, eps 1e-12).  One CTA per sequence; a lane owns G = d / 128 float4
// column groups of every row, warp w sums rows w * U + k + j * MP_WARPS * U (k < U: U rows loaded before they are added).
// The warps' partial sums meet in shared memory and are added in warp order: the bits depend on the tokens alone.
constexpr int MP_WARPS = 8;
template <int G>
__global__ void __launch_bounds__(MP_WARPS * 32)
mean_normalize_kernel(const float* __restrict__ x, const int32_t* __restrict__ seq_off, float* __restrict__ out, int ld_out)
{
    constexpr int D = G * 128, U = 16 / G < 4 ? 16 / G : 4;
    __shared__ __align__(16) float part[MP_WARPS][D];
    __shared__ float s_sq[MP_WARPS];
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t0 = seq_off[b], len = seq_off[b + 1] - t0;
    const float4* rows = reinterpret_cast<const float4*>(x + (size_t)t0 * D);
    float4 acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = make_float4(0.f, 0.f, 0.f, 0.f);
    auto add = [&](const float4& v, int g) { acc[g].x += v.x; acc[g].y += v.y; acc[g].z += v.z; acc[g].w += v.w; };
    int r0 = warp * U;
    for (; r0 + U <= len; r0 += MP_WARPS * U) {      // U whole rows: all U * G loads in flight before the adds
        float4 v[U][G];
#pragma unroll
        for (int k = 0; k < U; ++k)
#pragma unroll
            for (int g = 0; g < G; ++g) v[k][g] = rows[(size_t)(r0 + k) * (D / 4) + lane + 32 * g];
#pragma unroll
        for (int k = 0; k < U; ++k)
#pragma unroll
            for (int g = 0; g < G; ++g) add(v[k][g], g);
    }
#pragma unroll
    for (int k = 0; k < U; ++k)                      // the warp's last, partial step
        if (r0 + k < len)
#pragma unroll
            for (int g = 0; g < G; ++g) add(rows[(size_t)(r0 + k) * (D / 4) + lane + 32 * g], g);
#pragma unroll
    for (int g = 0; g < G; ++g) reinterpret_cast<float4*>(part[warp])[lane + 32 * g] = acc[g];
    __syncthreads();
    // thread i: float4 column group i (D / 4 <= 256 = the block size)
    const int c = threadIdx.x;
    const bool on = c < D / 4;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
    if (on) {
#pragma unroll
        for (int w = 0; w < MP_WARPS; ++w) {
            const float4 p = reinterpret_cast<const float4*>(part[w])[c];
            m.x += p.x; m.y += p.y; m.z += p.z; m.w += p.w;
        }
        const float fl = (float)len;
        m.x /= fl; m.y /= fl; m.z /= fl; m.w /= fl;
    }
    const float sq = warp_sum((m.x * m.x + m.y * m.y) + (m.z * m.z + m.w * m.w));
    if (lane == 0) s_sq[warp] = sq;
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < MP_WARPS; ++w) s += s_sq[w];
    const float n = fmaxf(sqrtf(s), 1e-12f);
    if (on) {
        float* o = out + (size_t)b * ld_out + 4 * c;
        o[0] = m.x / n; o[1] = m.y / n; o[2] = m.z / n; o[3] = m.w / n;
    }
}

// ------------------------------------------------------------------------ cross-encoder head
// BertForSequenceClassification with one label: score = act(w_c . tanh(W_p h + b_p) + b_c) over the [CLS] row h.  p holds
// W_p h + b_p (the pooler GEMM's output); one warp per pair, lane l adds elements l, l + 32, ... in order, then the butterfly
// of warp_sum: a fixed fp32 order, so a pair's score does not depend on the other pairs of the batch.
__global__ void __launch_bounds__(256)
classifier_head_kernel(const float* __restrict__ p, const float* __restrict__ w, const float* __restrict__ bias, int batch, int d,
                       int act, float* __restrict__ out)
{
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= batch) return;
    const float* row = p + (size_t)b * d;
    float s = 0.f;
    for (int i = lane; i < d; i += 32) s = fmaf(tanhf(row[i]), w[i], s);
    const float z = warp_sum(s) + bias[0];
    if (lane == 0) out[b] = act == EMB_ACT_SIGMOID ? 1.f / (1.f + expf(-z)) : z;
}

// Per query (one CTA): the top_k of its candidates' scores, descending, ties by fused position ascending.  Keys are
// (~ordered_bits(score)) << 32 | position: unique, so the ascending bitonic sort in shared memory gives one order whatever
// the sort does with equal keys.  Positions past the query's candidates are -1 with a NaN score.
constexpr int RS_MAX = 512;   // >= RERANK_MAX_CANDIDATES, a power of two
__global__ void __launch_bounds__(256)
rerank_select_kernel(const float* __restrict__ scores, const int32_t* __restrict__ pair_off, int top_k, int32_t* __restrict__ out_pos,
                     float* __restrict__ out_score)
{
    __shared__ uint64_t keys[RS_MAX];
    const int q = blockIdx.x;
    const int p0 = pair_off[q], n = pair_off[q + 1] - p0;
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) keys[i] = i < n ? make_key_desc(scores[p0 + i], (uint32_t)i) : KEY_PAD;
    __syncthreads();
    for (int k = 2; k <= n2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const uint64_t a = keys[i], c = keys[l];
                    if ((a > c) == ((i & k) == 0)) { keys[i] = c; keys[l] = a; }
                }
            }
            __syncthreads();
        }
    for (int i = threadIdx.x; i < top_k; i += blockDim.x) {
        const bool on = i < n;
        out_pos[(size_t)q * top_k + i] = on ? (int32_t)key_ordinal(keys[i]) : -1;
        out_score[(size_t)q * top_k + i] = on ? key_value_desc(keys[i]) : CUDART_NAN_F;
    }
}

// ------------------------------------------------------------------------------------ late interaction (ColBERT)
// MaxSim over a pair table: pair p scores the rows tab[p].rows [tab[p].n][dim] (stride dim; every row enters the max: the
// kept rows of a stored passage, or of a passage encoded in the call) against its query's q_rows unit vectors (rows of
// stride ld): score = sum_{i < q_rows} max_{j < n} q_i . d_j.  Query q owns pairs pair_off[q] .. pair_off[q + 1].  One CTA
// per (query, slice of its pairs): the query's rows are staged in shared memory once, then the CTA walks the 32-row chunks of
// its pairs as one sequence, with the next MS_STAGES - 1 chunks in flight by cp.async across pair boundaries.  Thread (i, jl)
// = (tid / 8, tid % 8) owns query row i and chunk rows jl + 8 u (u < 4): every dot product is one fp32 fmaf chain over
// k = 0 .. dim - 1 in order, the max over rows is exact (so the row order does not matter), and one thread adds the q_rows
// maxima in row order.  A pair's score therefore depends on its two token matrices alone, wherever its rows live.  Rows are
// padded by 4 floats in shared memory, so the 16-byte reads of 8 rows at one k hit 8 distinct bank groups.
struct MsPair { const float* rows; int32_t n, unused; };
constexpr int MS_QROWS = 32, MS_CHUNK = 32, MS_THREADS = 256, MS_STAGES = 3;
__global__ void __launch_bounds__(MS_THREADS)
maxsim_kernel(const float* __restrict__ qv, int q_rows, int ld, const MsPair* __restrict__ tab, const int32_t* __restrict__ pair_off,
              int dim, float* __restrict__ scores)
{
    extern __shared__ __align__(16) float ms_sm[];
    const int LDS = dim + 4, c4 = dim / 4;
    float* sQ = ms_sm;                                  // [MS_QROWS][LDS]
    float* sD = sQ + MS_QROWS * LDS;                    // [MS_STAGES][MS_CHUNK][LDS]
    float* sMax = sD + MS_STAGES * MS_CHUNK * LDS;      // [MS_QROWS]
    const int q = blockIdx.x, tid = threadIdx.x, i = tid >> 3, jl = tid & 7, step = (int)gridDim.y;
    const int p_end = pair_off[q + 1];
    int lp = pair_off[q] + (int)blockIdx.y, lc = 0;     // the next chunk to load: rows lc .. of pair lp
    if (lp >= p_end) return;
    MsPair lt = tab[lp];
    int cp = lp, cc = 0, cn = lt.n;                     // the chunk to score: rows cc .. of pair cp (cn rows)
    for (int x = tid; x < q_rows * c4; x += MS_THREADS) {
        const int r = x / c4, c = x - r * c4;
        *reinterpret_cast<float4*>(sQ + r * LDS + 4 * c) = *reinterpret_cast<const float4*>(qv + ((size_t)q * q_rows + r) * ld + 4 * c);
    }
    // one commit group per chunk slot, empty once the slice's chunks are all issued
    auto issue = [&](int stage) {
        if (lp < p_end) {
            const int n = lt.n - lc < MS_CHUNK ? lt.n - lc : MS_CHUNK;
            const float* src = lt.rows + (size_t)lc * dim;
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(sD + stage * MS_CHUNK * LDS);
            for (int x = tid; x < n * c4; x += MS_THREADS) {
                const int r = x / c4, c = x - r * c4;
                cp_async16_zfill(dst + 4u * (uint32_t)(r * LDS + 4 * c), src + 4 * (size_t)x, true);
            }
            lc += MS_CHUNK;
            if (lc >= lt.n) {
                lp += step; lc = 0;
                if (lp < p_end) lt = tab[lp];
            }
        }
        am_commit();
    };
#pragma unroll
    for (int s = 0; s < MS_STAGES - 1; ++s) issue(s);
    float m = -CUDART_INF_F;
    for (int t = 0; cp < p_end; ++t) {
        am_wait<MS_STAGES - 2>();
        __syncthreads();                                // chunk t (and the query rows) staged; chunk t - 1's stage consumed
        issue((t + MS_STAGES - 1) % MS_STAGES);
        const float* sC = sD + (t % MS_STAGES) * MS_CHUNK * LDS;
        const int n = cn - cc;                          // rows of this chunk: min(n, MS_CHUNK)
        if (i < q_rows) {
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            const float* qr = sQ + i * LDS;
            for (int k = 0; k < c4; ++k) {
                const float4 a = *reinterpret_cast<const float4*>(qr + 4 * k);
                const float4 b0 = *reinterpret_cast<const float4*>(sC + jl * LDS + 4 * k);
                const float4 b1 = *reinterpret_cast<const float4*>(sC + (jl + 8) * LDS + 4 * k);
                const float4 b2 = *reinterpret_cast<const float4*>(sC + (jl + 16) * LDS + 4 * k);
                const float4 b3 = *reinterpret_cast<const float4*>(sC + (jl + 24) * LDS + 4 * k);
                a0 = fmaf(a.x, b0.x, a0); a0 = fmaf(a.y, b0.y, a0); a0 = fmaf(a.z, b0.z, a0); a0 = fmaf(a.w, b0.w, a0);
                a1 = fmaf(a.x, b1.x, a1); a1 = fmaf(a.y, b1.y, a1); a1 = fmaf(a.z, b1.z, a1); a1 = fmaf(a.w, b1.w, a1);
                a2 = fmaf(a.x, b2.x, a2); a2 = fmaf(a.y, b2.y, a2); a2 = fmaf(a.z, b2.z, a2); a2 = fmaf(a.w, b2.w, a2);
                a3 = fmaf(a.x, b3.x, a3); a3 = fmaf(a.y, b3.y, a3); a3 = fmaf(a.z, b3.z, a3); a3 = fmaf(a.w, b3.w, a3);
            }
            if (jl < n) m = fmaxf(m, a0);
            if (jl + 8 < n) m = fmaxf(m, a1);
            if (jl + 16 < n) m = fmaxf(m, a2);
            if (jl + 24 < n) m = fmaxf(m, a3);
        }
        cc += MS_CHUNK;
        if (cc >= cn) {                                 // the pair's last chunk
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));   // the 8 threads of a query row are adjacent lanes
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
            if (jl == 0 && i < q_rows) sMax[i] = m;
            __syncthreads();
            if (tid == 0) {
                float s = 0.f;
                for (int r = 0; r < q_rows; ++r) s += sMax[r];
                scores[cp] = s;
            }
            m = -CUDART_INF_F;
            cp += step; cc = 0;
            if (cp < p_end) cn = tab[cp].n;
        }
    }
    am_wait<0>();
}
static size_t maxsim_smem(int dim) { return sizeof(float) * ((size_t)(MS_QROWS + MS_STAGES * MS_CHUNK) * (dim + 4) + MS_QROWS); }

// Row r of the output, dst[r] (dim floats), is row src[r] of `in` (stride ld): the kept rows of passages encoded at stride
// li_pad, gathered into a store's slabs or a call's compact scratch.  One warp per row; a copy, so the bits do not change.
__global__ void __launch_bounds__(256)
late_gather_kernel(const float* __restrict__ in, int ld, const int32_t* __restrict__ src, float* const* __restrict__ dst, int n_rows, int dim)
{
    const int r = (int)((blockIdx.x * 256u + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (r >= n_rows) return;
    const float4* a = reinterpret_cast<const float4*>(in + (size_t)src[r] * ld);
    float4* b = reinterpret_cast<float4*>(dst[r]);
    for (int c = lane; c < dim / 4; c += 32) b[c] = a[c];
}

// ------------------------------------------------------------------------------------ host
// launch with programmatic stream serialization (see pdl_wait in tc_ptx.cuh); only for kernels that call pdl_wait()
template <typename... KArgs, typename... Args>
static void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    KRAG_CUDA(cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
    count_launch();
}

template <int DH, int WARPS, int KB, int STAGES, int PLANES, bool REL, bool KVL>
static void launch_attention_mma(const uint16_t* q_hi, const uint16_t* q_lo, const int32_t* seq_off, uint16_t* out_hi, uint16_t* out_lo, int d,
                                 int heads, int batch, int max_len, bool first_rows, const float* rel_tab, const int32_t* kv_len, cudaStream_t st)
{
    using Cfg = AmCfg<DH, WARPS, KB, STAGES, PLANES>;
    constexpr size_t smem = Cfg::SMEM + (REL ? sizeof(float) * REL_TAB : 0);
    static bool attr_set = false;
    if (!attr_set) {
        KRAG_CUDA(cudaFuncSetAttribute(attention_mma_kernel<DH, WARPS, KB, STAGES, PLANES, REL, KVL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    const unsigned q_blocks = first_rows ? 1u : (unsigned)((max_len + 16 * WARPS - 1) / (16 * WARPS));
    launch_pdl(attention_mma_kernel<DH, WARPS, KB, STAGES, PLANES, REL, KVL>, dim3(q_blocks, (unsigned)heads, (unsigned)batch),
               dim3(WARPS * 32), smem, st, q_hi, q_lo, seq_off, out_hi, out_lo, d, heads, rel_tab, kv_len);
}
template <int DH, int PLANES, bool REL, bool KVL>
static void attention_mma_blocks(const uint16_t* q_hi, const uint16_t* q_lo, const int32_t* seq_off, uint16_t* out_hi, uint16_t* out_lo, int d,
                                 int heads, int batch, int max_len, bool first_rows, const float* rel_tab, const int32_t* kv_len, cudaStream_t st)
{
    if constexpr (KVL) {                   // the late-interaction forward's blocking (encoder_forward: max_len > 64)
        launch_attention_mma<DH, 4, 64, 2, PLANES, REL, KVL>(q_hi, q_lo, seq_off, out_hi, out_lo, d, heads, batch, max_len, first_rows, rel_tab, kv_len, st);
    } else if (max_len <= 32)
        launch_attention_mma<DH, 2, 32, 1, PLANES, REL, KVL>(q_hi, q_lo, seq_off, out_hi, out_lo, d, heads, batch, max_len, first_rows, rel_tab, kv_len, st);
    else if (max_len <= 64)
        launch_attention_mma<DH, 4, 64, 1, PLANES, REL, KVL>(q_hi, q_lo, seq_off, out_hi, out_lo, d, heads, batch, max_len, first_rows, rel_tab, kv_len, st);
    else launch_attention_mma<DH, 4, 64, 2, PLANES, REL, KVL>(q_hi, q_lo, seq_off, out_hi, out_lo, d, heads, batch, max_len, first_rows, rel_tab, kv_len, st);
}
// queries (<= 32 tokens): 2 warps, one key block; <= 64: 4 warps, one block; chunks: 4 warps, 64-key blocks, double-buffered.
// first_rows: only the first block of query rows of every sequence (the [CLS] row among them); a query row's result does
// not depend on which other rows run, and the key blocking follows max_len either way.  PLANES == 1: q_lo / out_lo are not used.
// rel_tab: the MPNet relative-position bias table (REL instantiations), null for BERT.  kv_len: per-sequence key counts
// (device, KVL instantiations; BERT only), null: every row is a key.
template <int DH, int PLANES>
static void attention_mma(const uint16_t* q_hi, const uint16_t* q_lo, const int32_t* seq_off, uint16_t* out_hi, uint16_t* out_lo, int d, int heads,
                          int batch, int max_len, bool first_rows, const float* rel_tab, const int32_t* kv_len, cudaStream_t st)
{
    if (rel_tab && kv_len) throw std::runtime_error("embedder: key lengths are not combined with the relative-position bias");
    if (rel_tab) attention_mma_blocks<DH, PLANES, true, false>(q_hi, q_lo, seq_off, out_hi, out_lo, d, heads, batch, max_len, first_rows, rel_tab, nullptr, st);
    else if (kv_len) attention_mma_blocks<DH, PLANES, false, true>(q_hi, q_lo, seq_off, out_hi, out_lo, d, heads, batch, max_len, first_rows, nullptr, kv_len, st);
    else attention_mma_blocks<DH, PLANES, false, false>(q_hi, q_lo, seq_off, out_hi, out_lo, d, heads, batch, max_len, first_rows, nullptr, nullptr, st);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn emb_encode()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
// 2D map over one split plane [rows, cols] of fp16, box = 64 halfs (one 128-byte swizzle row) x box_rows
static void emb_map(CUtensorMap* tm, const uint16_t* base, int rows, int cols, int box_rows = GM_TILE)
{
    EncodeTiledFn enc = emb_encode();
    if (!enc) throw CudaError{cudaErrorUnknown, "cuTensorMapEncodeTiled unavailable", __FILE__, __LINE__};
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};
    cuuint32_t box[2] = {(cuuint32_t)GH_KB, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    if (enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<uint16_t*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        throw CudaError{cudaErrorUnknown, "cuTensorMapEncodeTiled failed", __FILE__, __LINE__};
}

template <int BN, int PLANES, int EP>
static void launch_gemm_ep(dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& tmA1, const CUtensorMap& tmA2, const CUtensorMap& tmB1,
                           const CUtensorMap& tmB2, int M, int N, int splits, int kb_per_split, int n_stages, int b_evict_first,
                           const float* bias, const float* residual, bool gelu, const GemmOut& out, float* ws, const EpiArgs& ep)
{
    static bool attr = false;
    if (!attr) { KRAG_CUDA(cudaFuncSetAttribute(gemm_f16s_kernel<BN, PLANES, EP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
    launch_pdl(gemm_f16s_kernel<BN, PLANES, EP>, grid, dim3(GM_THREADS), smem, st, tmA1, tmA2, tmB1, tmB2, M, N, splits, kb_per_split,
               n_stages, b_evict_first, bias, residual, gelu ? 1 : 0, out, ws, ep);
}
// gemm_f16s_kernel over the 128 x BN tiles of C and `splits` K slices, min(work items, SMs) persistent CTAs
template <int BN, int PLANES>
static void launch_gemm(const DeviceInfo& di, const SplitMat& A, const SplitMat& B, int M, int N, int K, int splits, const float* bias,
                        const float* residual, bool gelu, const GemmOut& out, float* ws, cudaStream_t st, const EpiArgs& ep)
{
    constexpr int stage_bytes = PLANES * (GM_SLAB + BN * 128);
    constexpr int n_stages = GM_SMEM_BUDGET / stage_bytes < GM_MAX_STAGES ? GM_SMEM_BUDGET / stage_bytes : GM_MAX_STAGES;
    constexpr size_t smem = 1024 + (size_t)n_stages * stage_bytes + 2 * GM_MAX_STAGES * 8;
    CUtensorMap tmA1, tmA2, tmB1, tmB2;
    emb_map(&tmA1, A.hi, M, K); emb_map(&tmA2, PLANES == 2 ? A.lo : A.hi, M, K);     // PLANES == 1: the second maps are not read
    emb_map(&tmB1, B.hi, N, K, BN); emb_map(&tmB2, PLANES == 2 ? B.lo : B.hi, N, K, BN);
    const int m_tiles = (M + GM_TILE - 1) / GM_TILE;
    const int total = m_tiles * (N / BN) * splits;
    const int grid = total < di.sm_count ? total : di.sm_count;
    // one activation tile: every weight byte is read once, keep it out of the way of the activations in L2
    const int kbs = K / GH_KB / splits, evict_b = m_tiles == 1 ? 1 : 0;
    if (ep.mode == EP_ROPE)
        launch_gemm_ep<BN, PLANES, EP_ROPE>(dim3((unsigned)grid), smem, st, tmA1, tmA2, tmB1, tmB2, M, N, splits, kbs, n_stages, evict_b, bias,
                                            residual, gelu, out, ws, ep);
    else if (ep.mode == EP_SWIGLU)
        launch_gemm_ep<BN, PLANES, EP_SWIGLU>(dim3((unsigned)grid), smem, st, tmA1, tmA2, tmB1, tmB2, M, N, splits, kbs, n_stages, evict_b, bias,
                                              residual, gelu, out, ws, ep);
    else
        launch_gemm_ep<BN, PLANES, EP_PLAIN>(dim3((unsigned)grid), smem, st, tmA1, tmA2, tmB1, tmB2, M, N, splits, kbs, n_stages, evict_b, bias,
                                             residual, gelu, out, ws, ep);
}

// Tile width and K split of a linear layer of M rows.  Every output element is summed in an order fixed by (bn, splits)
// alone, so a plan made for M rows computes the same bits on any subset of those rows.
GemmPlan linear_plan(const DeviceInfo& di, int M, int N, int K, bool ln, bool have_ws, size_t ws_floats, int planes)
{
    const int m_tiles = (M + GM_TILE - 1) / GM_TILE;
    const int tiles128 = m_tiles * (N / GM_TILE);
    if (have_ws && tiles128 < di.sm_count / 2 && N % 64 == 0 && K % GH_KB == 0 && (!ln || N <= 1024)) {
        // long-K layers over several activation tiles (FFN2 for tens of queries): 128 x 128 tiles halve the operand
        // re-reads through L2 (the binding resource); split-K restores the CTA count
        const int BN = m_tiles == 1 ? 32 : ((K >= 2048 && N % 128 == 0) ? 128 : 64);
        const int ctas = m_tiles * (N / BN), kblocks = K / GH_KB;
        int splits = 1;
        if (ctas <= di.sm_count / 3) {              // 72 CTAs with the whole K range beat 144 + a reduce kernel
            const int want = di.sm_count / ctas < SK_MAX_SPLITS ? di.sm_count / ctas : SK_MAX_SPLITS;
            for (int sp = want; sp >= 2; --sp)
                if (kblocks % sp == 0 && kblocks / sp >= 2 && (size_t)sp * M * N <= ws_floats) { splits = sp; break; }
        }
        return GemmPlan{BN, splits, true};
    }
    // single-plane product: one accumulator per thread leaves room for 128 x 256 tiles.  Taken from two waves of them on:
    // at 8192 rows they measured 2-13% faster than 128 x 128 for N = 1536 ... 3072 and 7-9% slower for N = 768, where 192
    // tiles leave half of the second wave's SMs idle (DESIGN.md section 4, "Cross-encoder head")
    if (planes == 1 && N % 256 == 0 && m_tiles * (N / 256) >= 2 * di.sm_count) return GemmPlan{256, 1, false};
    return GemmPlan{128, 1, false};
}

// Linear layer on split operands: C = A . B^T + bias (+GELU) (+residual) -> fp32 C and / or split planes of C; with ln_g the
// row LayerNorm of that goes to Y (fp32) and its split planes (C is then scratch).  plan: null = linear_plan(M, ...).
void launch_linear(const DeviceInfo& di, const SplitMat& A, const SplitMat& B, int M, int N, int K, const float* bias, const float* residual,
                   bool gelu, float* C, uint16_t* C_hi, uint16_t* C_lo, const float* ln_g, const float* ln_b, float eps, float* Y,
                   uint16_t* Y_hi, uint16_t* Y_lo, float* ws, size_t ws_floats, cudaStream_t st, const GemmPlan* plan, int planes,
                   const EpiArgs* epi)
{
    if (ln_g && N > 32 * LN_MAX_GROUPS * 8) throw std::runtime_error("launch_linear: fused LayerNorm rows hold at most 1024 elements");
    const EpiArgs ep = epi ? *epi : EpiArgs{EP_PLAIN, nullptr, nullptr, 0, 0};
    if (ep.mode != EP_PLAIN && (ln_g || residual || gelu))
        throw std::runtime_error("launch_linear: the rotary and gated epilogues take no LayerNorm, residual or GELU");
    const GemmPlan p = plan ? *plan : linear_plan(di, M, N, K, ln_g != nullptr, ws != nullptr, ws_floats, planes);
    if (planes == 1) { C_lo = nullptr; Y_lo = nullptr; }
    if (planes != 1 && planes != 2) throw std::runtime_error("launch_linear: one or two operand planes");
    if (N % p.bn || (p.bn == 256 && planes != 1) || K % GH_KB || (K / GH_KB) % p.splits || (p.splits > 1 && (!ws || (size_t)p.splits * M * N > ws_floats)))
        throw std::runtime_error("launch_linear: plan does not fit the problem");
    if (p.small_m) {
        // splits == 1 and a LayerNorm to follow: the GEMM writes fp32 C (scratch), the LayerNorm kernel writes Y + planes
        const GemmOut direct = ln_g ? GemmOut{C, nullptr, nullptr} : GemmOut{C, C_hi, C_lo};
        if (planes == 1) {
            if (p.bn == 32) launch_gemm<32, 1>(di, A, B, M, N, K, p.splits, bias, residual, gelu, direct, ws, st, ep);
            else if (p.bn == 256) launch_gemm<256, 1>(di, A, B, M, N, K, p.splits, bias, residual, gelu, direct, ws, st, ep);
            else if (p.bn == 128) launch_gemm<128, 1>(di, A, B, M, N, K, p.splits, bias, residual, gelu, direct, ws, st, ep);
            else launch_gemm<64, 1>(di, A, B, M, N, K, p.splits, bias, residual, gelu, direct, ws, st, ep);
        } else if (p.bn == 32) launch_gemm<32, 2>(di, A, B, M, N, K, p.splits, bias, residual, gelu, direct, ws, st, ep);
        else if (p.bn == 128) launch_gemm<128, 2>(di, A, B, M, N, K, p.splits, bias, residual, gelu, direct, ws, st, ep);
        else launch_gemm<64, 2>(di, A, B, M, N, K, p.splits, bias, residual, gelu, direct, ws, st, ep);
        if (p.splits > 1) {
            auto reduce = ep.mode == EP_ROPE ? splitk_reduce_kernel<EP_ROPE>
                          : ep.mode == EP_SWIGLU ? splitk_reduce_kernel<EP_SWIGLU> : splitk_reduce_kernel<EP_PLAIN>;
            launch_pdl(reduce, dim3((unsigned)M), dim3(256), 0, st, ws, p.splits, M, N, bias, residual, gelu ? 1 : 0, ln_g, ln_b,
                       eps, ln_g ? Y : C, ln_g ? Y_hi : C_hi, ln_g ? Y_lo : C_lo, ep);
            return;
        }
    } else {
        const GemmOut direct = ln_g ? GemmOut{C, nullptr, nullptr} : GemmOut{C, C_hi, C_lo};
        if (planes == 1 && p.bn == 256) launch_gemm<256, 1>(di, A, B, M, N, K, 1, bias, residual, gelu, direct, nullptr, st, ep);
        else if (planes == 1) launch_gemm<128, 1>(di, A, B, M, N, K, 1, bias, residual, gelu, direct, nullptr, st, ep);
        else launch_gemm<128, 2>(di, A, B, M, N, K, 1, bias, residual, gelu, direct, nullptr, st, ep);
    }
    if (ln_g) {
        launch_pdl(layernorm_kernel, dim3((unsigned)((M * 32 + 255) / 256)), dim3(256), 0, st, C, Y, Y_hi, Y_lo, ln_g, ln_b, M, N, eps);
    }
}

// test hook (krag_debug_gemm_tf32 / krag_debug_linear_ln): fp32 device operands are split here, then take the product path
void launch_linear_f32(const DeviceInfo& di, const float* A, const float* B, int M, int N, int K, const float* bias, const float* residual,
                       bool gelu, float* C, const float* ln_g, const float* ln_b, float eps, float* Y, float* ws, size_t ws_floats,
                       cudaStream_t st, int tile_n, int reps, float* ms, int planes)
{
    if (tile_n != 0 && tile_n != 32 && tile_n != 64 && tile_n != 128 && !(tile_n == 256 && planes == 1))
        throw std::runtime_error("launch_linear_f32: tile width must be 0, 32, 64 or 128 (256: single-plane product only)");
    const GemmPlan forced{tile_n, 1, true};
    const GemmPlan* plan = tile_n ? &forced : nullptr;
    const size_t na = (size_t)M * K, nb = (size_t)N * K;
    DevArray<uint16_t> buf;
    buf.alloc((int64_t)(2 * na + 2 * nb));
    SplitMat As{buf.p, buf.p + na}, Bs{buf.p + 2 * na, buf.p + 2 * na + nb};
    launch_split_f16(A, As.hi, As.lo, (int64_t)na, st);
    launch_split_f16(B, Bs.hi, Bs.lo, (int64_t)nb, st);
    auto run = [&] {
        launch_linear(di, As, Bs, M, N, K, bias, residual, gelu, C, nullptr, nullptr, ln_g, ln_b, eps, Y, nullptr, nullptr, ws, ws_floats, st, plan, planes);
    };
    run();
    if (reps > 0) {
        // C = A.B^T + bias (+residual) does not read C: repeating the launch leaves the result as it was
        cudaEvent_t e0, e1;
        KRAG_CUDA(cudaEventCreate(&e0));
        KRAG_CUDA(cudaEventCreate(&e1));
        KRAG_CUDA(cudaEventRecord(e0, st));
        for (int r = 0; r < reps; ++r) run();
        KRAG_CUDA(cudaEventRecord(e1, st));
        KRAG_CUDA(cudaEventSynchronize(e1));
        float t = 0.f;
        KRAG_CUDA(cudaEventElapsedTime(&t, e0, e1));
        cudaEventDestroy(e0); cudaEventDestroy(e1);
        if (ms) *ms = t / (float)reps;
    }
    KRAG_CUDA(cudaStreamSynchronize(st));
}


struct Embedder {
    DeviceInfo di;
    BertConfig cfg;
    std::map<std::string, DevArray<float>> t;   // HF tensor name -> device copy
    std::vector<DevArray<float>> bqkv;          // fused Q|K|V bias per layer (finalize)
    // split fp16 planes of the GEMM weights (finalize): per layer QKV (fused), attention output, FFN1, FFN2
    std::vector<SplitMat> s_qkv, s_o, s_f1, s_f2;
    std::vector<DevArray<uint16_t>> planes;     // the buffers all weight planes live in
    SplitMat s_pool{nullptr, nullptr};          // pooler.dense.weight (cross-encoders: finalize found the classifier head)
    DevArray<float> rel_tab;                    // MPNet: [heads][REL_TAB] relative-position bias by distance (finalize); else null
    // rotary encoders (nomic-bert): rope_base > 0 (krag_embedder_set_rotary); finalize permutes each head's Q and K weight rows
    // so that elements i and i + dh/2 are adjacent and builds rope [max_pos][dh/2] (cos, sin)
    float rope_base = 0.f;
    DevArray<float> rope;
    // gated FFN (SwiGLU): loaded with intermediate.gate.*; finalize interleaves up / gate rows into s_f1 and their biases into bf1
    bool gated = false;
    std::vector<DevArray<float>> bf1;
    bool has_head = false;
    // late interaction (ColBERT): li_dim > 0 (krag_embedder_set_late_interaction); finalize splits linear.weight [li_dim][hidden]
    // zero-padded to li_pad = the next multiple of 128 rows (the padded outputs are exact zeros), li_bias is li_pad zeros
    int li_dim = 0, li_pad = 0;
    SplitMat s_li{nullptr, nullptr};
    DevArray<float> li_bias;
    DevArray<float> li_c, li_q, li_p;     // projection scratch [cap_tok][li_pad]; query / passage unit vectors, rows of li_pad
    DevArray<float> li_k;                 // the kept rows of a call's passages, rows of li_dim (late_gather_kernel)
    DevArray<int32_t> d_kvl, li_src;      // li_src / li_dst: a gather's source row and destination of every kept row
    DevArray<float*> li_dst;
    DevArray<MsPair> li_tab;              // maxsim_kernel's pair table
    // stores of passage vectors (LateStore) made from this embedder: their slabs share one budget of device bytes
    int64_t store_budget = 0, store_bytes = 0;
    int n_stores = 0;
    bool finalized = false;
    cudaStream_t st = nullptr;
    cudaEvent_t done = nullptr, in_ev = nullptr;
    // captured forward per (n_tok, batch, max_len, cls_rows, head, precision, late): head = 1 for cross-encoder pairs (token
    // types uploaded); the two precisions run different kernels; late = 1 for a late-interaction forward, 2 with key lengths
    using GraphKey = std::tuple<int, int, int, int, int, int, int>;
    std::map<GraphKey, cudaGraphExec_t> graphs;
    std::map<GraphKey, int> seen;
    int precision = EMB_PREC_FP32;        // EMB_PREC_FP16: single-plane products (the hi planes of weights and activations)
    int pooling = EMB_POOL_CLS;           // read by the final writer, which runs outside the captured graphs
    int pos_off = 0;                      // position row of a sequence's first token: built into the host's position array,
                                          // which is uploaded before a graph launches, so no captured pointer or shape depends on it
    bool cls_rows_only = true;            // CLS pooling: the last layer after QKV + attention runs on the [CLS] rows only
    // workspaces, grown on demand
    int cap_tok = 0, cap_batch = 0;
    DevArray<int32_t> d_tok, d_pos, d_off, d_typ;
    // reranking: one score per pair of a call, the per-query pair offsets, the selected positions | scores
    DevArray<float> scores;
    DevArray<int32_t> d_poff, sel;
    DevArray<float> x, x2, out;
    DevArray<uint16_t> xs, cs, fs;        // split planes [2][T][*] of x (LayerNorm outputs), attention context, FFN1 output
    DevArray<uint16_t> qkv;               // split planes [2][n_tok][3d] of the QKV projection (the lo plane starts at n_tok rows)
    DevArray<float> ws;                   // split-K partials (small token counts)
    // the last layer on the [CLS] rows only: residual stream, GEMM scratch, split planes of the attention context, of the
    // LayerNorm output and of FFN1's output, [cap_batch] rows each
    DevArray<float> cx, cx2;
    DevArray<uint16_t> ccs, cxs, cfs;
    static constexpr size_t WS_FLOATS = (size_t)4 << 20;

    void drop_graphs()
    {
        for (auto& kv : graphs) cudaGraphExecDestroy(kv.second);
        graphs.clear();
    }
    ~Embedder()
    {
        drop_graphs();
        if (done) cudaEventDestroy(done);
        if (in_ev) cudaEventDestroy(in_ev);
        if (st) cudaStreamDestroy(st);
    }
};

// the device copy of a loaded tensor, which must hold exactly n elements: the kernels index it by the config's sizes
// (embed_ln_kernel clamps token ids to cfg.vocab, not to the rows uploaded)
static float* emb_get(Embedder* e, const std::string& name, int64_t n)
{
    auto it = e->t.find(name);
    if (it == e->t.end() || it->second.p == nullptr) throw std::runtime_error("embedder: tensor not loaded: " + name);
    if (it->second.cap != n)
        throw std::runtime_error("embedder: " + name + " must hold " + std::to_string(n) + " elements (the config's shape), not " +
                                 std::to_string(it->second.cap));
    return it->second.p;
}
static std::string lname(int l, const char* s) { return "encoder.layer." + std::to_string(l) + "." + s; }

Embedder* embedder_create(const DeviceInfo& di, const BertConfig& cfg)
{
    if (cfg.hidden % 128 || cfg.inter % 128 || cfg.hidden % cfg.heads || cfg.hidden / cfg.heads > 64 || (cfg.hidden / cfg.heads) % 32 || cfg.hidden > 1024)
        throw std::runtime_error("embedder: hidden/intermediate must be multiples of 128, hidden <= 1024 and head_dim 32 or 64");
    auto e = std::make_unique<Embedder>();
    e->di = di; e->cfg = cfg;
    KRAG_CUDA(cudaStreamCreateWithFlags(&e->st, cudaStreamNonBlocking));
    return e.release();
}

void embedder_load(Embedder* e, const char* name, const float* data, int64_t n)
{
    DevArray<float> p;
    p.alloc(n);
    KRAG_CUDA(cudaMemcpy(p.p, data, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice));
    e->t[name] = std::move(p);
    e->finalized = false;
}

static SplitMat emb_split_weight(Embedder* e, const float* w, size_t n)
{
    DevArray<uint16_t> p;
    p.alloc((int64_t)(2 * n));
    SplitMat m{p.p, p.p + n};
    e->planes.push_back(std::move(p));
    launch_split_f16(w, m.hi, m.lo, (int64_t)n, e->st);
    return m;
}

// MPNetEncoder.relative_position_bucket(rel, num_buckets = 32, max_distance = 128): future keys (rel > 0) take 16 + b(rel),
// the others b(-rel); b(n) = n below 8, else min(15, 8 + floor(ln(n / 8) / ln 16 * 8)).  b saturates from n = 91 on, so the
// kernel's clamp of the distance to +-REL_MAX changes no bucket at any sequence length.
int relative_bucket(int rel)
{
    rel = rel < -REL_MAX ? -REL_MAX : (rel > REL_MAX ? REL_MAX : rel);
    const int base = rel > 0 ? 16 : 0, n = rel > 0 ? rel : -rel;
    if (n < 8) return base + n;
    const int v = 8 + (int)(std::log(n / 8.0) / std::log(16.0) * 8.0);
    return base + (v < 15 ? v : 15);
}
static const char* const REL_BIAS = "encoder.relative_attention_bias.weight";   // MPNet: [32 buckets][heads]
static const char* const LI_WEIGHT = "linear.weight";                           // ColBERT: [dim][hidden], no bias
constexpr int REL_BUCKETS = 32;

// transformers' default RoPE (NomicBertRotaryEmbedding): inv_freq[i] = 1 / base^(2i / dh) and the angle fp32(pos) *
// inv_freq[i], both fp32 as torch computes them; cos and sin of that fp32 angle rounded to fp32.  (Angles computed in fp64
// would differ by up to half an fp32 ulp of the angle: 2.4e-4 rad at position 8000.)
void rotary_cos_sin(float base, int dh, int pos, float* cos_out, float* sin_out)
{
    for (int i = 0; i < dh / 2; ++i) {
        const float ex = (float)(2 * i) / (float)dh;
        const float inv = 1.f / (float)std::pow((double)base, (double)ex);
        const float theta = (float)pos * inv;
        cos_out[i] = (float)std::cos((double)theta);
        sin_out[i] = (float)std::sin((double)theta);
    }
}

void embedder_set_late_interaction(Embedder* e, int dim, const float* weight, int64_t n)
{
    if (dim < 16 || dim > 256 || dim % 16)
        throw std::runtime_error("embedder: the late-interaction dim must be a multiple of 16 in [16, 256]");
    if (n != (int64_t)dim * e->cfg.hidden)
        throw std::runtime_error(std::string("embedder: ") + LI_WEIGHT + " must hold dim x hidden = " + std::to_string((int64_t)dim * e->cfg.hidden) +
                                 " elements, not " + std::to_string(n));
    embedder_load(e, LI_WEIGHT, weight, n);
    e->li_dim = dim;
}

void embedder_set_rotary(Embedder* e, float base)
{
    if (!(base >= 0.f) || std::isinf(base)) throw std::runtime_error("embedder: the rotary base must be finite and >= 0 (0: off)");
    e->rope_base = base;
    e->finalized = false;
}

static bool emb_has(const Embedder* e, const std::string& name)
{
    const auto it = e->t.find(name);
    return it != e->t.end() && it->second.p;
}
// rows [heads * dh][cols] copied to dst with each head's rows i and i + dh/2 made adjacent (rows 2i, 2i + 1): the pair the
// rotary epilogue rotates is then one thread's two columns (q . k is unchanged when Q and K are permuted alike)
static void rope_permute_rows(float* dst, const float* src, int heads, int dh, int cols, cudaStream_t st)
{
    const int half = dh / 2;
    const size_t row = sizeof(float) * (size_t)cols;
    for (int h = 0; h < heads; ++h)
        for (int s = 0; s < 2; ++s)
            KRAG_CUDA(cudaMemcpy2DAsync(dst + ((size_t)h * dh + s) * cols, 2 * row, src + ((size_t)h * dh + (size_t)s * half) * cols, row, row,
                                        (size_t)half, cudaMemcpyDeviceToDevice, st));
}
// up rows 8b .. 8b + 7 -> rows 16b .. 16b + 7 and gate rows 8b .. 8b + 7 -> rows 16b + 8 .. 16b + 15 of dst [2 * inter][cols]
static void swiglu_interleave_rows(float* dst, const float* up, const float* gate, int inter, int cols, cudaStream_t st)
{
    const size_t blk = sizeof(float) * 8 * (size_t)cols;
    KRAG_CUDA(cudaMemcpy2DAsync(dst, 2 * blk, up, blk, blk, (size_t)inter / 8, cudaMemcpyDeviceToDevice, st));
    KRAG_CUDA(cudaMemcpy2DAsync(dst + 8 * (size_t)cols, 2 * blk, gate, blk, blk, (size_t)inter / 8, cudaMemcpyDeviceToDevice, st));
}

void embedder_finalize(Embedder* e)
{
    const int d = e->cfg.hidden, inter = e->cfg.inter;
    e->finalized = false;
    e->bqkv.clear(); e->planes.clear(); e->s_qkv.clear(); e->s_o.clear(); e->s_f1.clear(); e->s_f2.clear();
    e->s_pool = SplitMat{nullptr, nullptr}; e->has_head = false;
    e->rel_tab.release(); e->rope.release(); e->bf1.clear(); e->gated = false;
    e->s_li = SplitMat{nullptr, nullptr}; e->li_pad = 0; e->li_bias.release();
    e->drop_graphs(); e->seen.clear();   // captured weight pointers are about to change
    const BertConfig& c = e->cfg;
    const int dh = d / c.heads;
    // every size first: a refused state leaves no half-built planes behind
    const auto rit = e->t.find(REL_BIAS);
    const bool rel = rit != e->t.end() && rit->second.p;   // an MPNet encoder: loaded with the relative-position bias
    if (rel) emb_get(e, REL_BIAS, (int64_t)REL_BUCKETS * c.heads);
    if (e->li_dim) emb_get(e, LI_WEIGHT, (int64_t)e->li_dim * d);
    const bool rotary = e->rope_base > 0.f;
    // a gated FFN: every layer loaded with intermediate.gate.weight [inter][hidden] (and its bias), or none
    const bool gated = emb_has(e, lname(0, "intermediate.gate.weight"));
    for (int l = 0; l < c.layers; ++l) {
        if (emb_has(e, lname(l, "intermediate.gate.weight")) != gated)
            throw std::runtime_error("embedder: " + lname(l, "intermediate.gate.weight") + (gated ? " missing" : " loaded") +
                                     ": a gated FFN needs the gate tensors on every layer (" + lname(0, "intermediate.gate.weight") +
                                     (gated ? " is loaded)" : " is not)"));
        if (gated) { emb_get(e, lname(l, "intermediate.gate.weight"), (int64_t)inter * d); emb_get(e, lname(l, "intermediate.gate.bias"), inter); }
    }
    emb_get(e, "embeddings.word_embeddings.weight", (int64_t)c.vocab * d);
    if (!rotary) emb_get(e, "embeddings.position_embeddings.weight", (int64_t)c.max_pos * d);
    emb_get(e, "embeddings.token_type_embeddings.weight", (int64_t)c.type_vocab * d);
    emb_get(e, "embeddings.LayerNorm.weight", d); emb_get(e, "embeddings.LayerNorm.bias", d);
    for (int l = 0; l < c.layers; ++l) {
        for (const char* nm : {"attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"}) {
            emb_get(e, lname(l, nm) + ".weight", (int64_t)d * d); emb_get(e, lname(l, nm) + ".bias", d);
        }
        for (const char* nm : {"attention.output.LayerNorm.weight", "attention.output.LayerNorm.bias", "output.dense.bias",
                               "output.LayerNorm.weight", "output.LayerNorm.bias"})
            emb_get(e, lname(l, nm), d);
        emb_get(e, lname(l, "intermediate.dense.weight"), (int64_t)inter * d); emb_get(e, lname(l, "intermediate.dense.bias"), inter);
        emb_get(e, lname(l, "output.dense.weight"), (int64_t)d * inter);
    }
    DevArray<float> wtmp;
    wtmp.alloc(gated && 2 * inter > 3 * d ? (int64_t)2 * inter * d : (int64_t)3 * d * d);
    for (int l = 0; l < e->cfg.layers; ++l) {
        DevArray<float> b;
        b.alloc((int64_t)3 * d);
        const char* names[3] = {"attention.self.query", "attention.self.key", "attention.self.value"};
        for (int j = 0; j < 3; ++j) {
            const float* w = emb_get(e, lname(l, names[j]) + ".weight", (int64_t)d * d);
            const float* bj = emb_get(e, lname(l, names[j]) + ".bias", d);
            if (rotary && j < 2) {                       // Q and K: each head's (i, i + dh/2) rows adjacent
                rope_permute_rows(wtmp.p + (size_t)j * d * d, w, c.heads, dh, d, e->st);
                rope_permute_rows(b.p + (size_t)j * d, bj, c.heads, dh, 1, e->st);
                continue;
            }
            KRAG_CUDA(cudaMemcpyAsync(wtmp.p + (size_t)j * d * d, w, sizeof(float) * (size_t)d * d, cudaMemcpyDeviceToDevice, e->st));
            KRAG_CUDA(cudaMemcpyAsync(b.p + (size_t)j * d, bj, sizeof(float) * (size_t)d, cudaMemcpyDeviceToDevice, e->st));
        }
        e->bqkv.push_back(std::move(b));
        e->s_qkv.push_back(emb_split_weight(e, wtmp.p, (size_t)3 * d * d));       // stream order: the split reads wtmp before the next layer overwrites it
        e->s_o.push_back(emb_split_weight(e, emb_get(e, lname(l, "attention.output.dense.weight"), (int64_t)d * d), (size_t)d * d));
        if (gated) {                                     // FFN1 = [up; gate] rows interleaved in blocks of 8, N = 2 * inter
            DevArray<float> bf;
            bf.alloc((int64_t)2 * inter);
            swiglu_interleave_rows(wtmp.p, emb_get(e, lname(l, "intermediate.dense.weight"), (int64_t)inter * d),
                                   emb_get(e, lname(l, "intermediate.gate.weight"), (int64_t)inter * d), inter, d, e->st);
            swiglu_interleave_rows(bf.p, emb_get(e, lname(l, "intermediate.dense.bias"), inter), emb_get(e, lname(l, "intermediate.gate.bias"), inter),
                                   inter, 1, e->st);
            e->bf1.push_back(std::move(bf));
            e->s_f1.push_back(emb_split_weight(e, wtmp.p, (size_t)2 * inter * d));
        } else {
            e->s_f1.push_back(emb_split_weight(e, emb_get(e, lname(l, "intermediate.dense.weight"), (int64_t)inter * d), (size_t)inter * d));
        }
        e->s_f2.push_back(emb_split_weight(e, emb_get(e, lname(l, "output.dense.weight"), (int64_t)d * inter), (size_t)d * inter));
    }
    if (rotary) {
        // (cos, sin) by [position][pair]: ~2 MB at 8192 positions x 32 pairs
        const int half = dh / 2;
        std::vector<float> tab((size_t)c.max_pos * half * 2), cs((size_t)half), sn((size_t)half);
        for (int p = 0; p < c.max_pos; ++p) {
            rotary_cos_sin(e->rope_base, dh, p, cs.data(), sn.data());
            for (int i = 0; i < half; ++i) { tab[((size_t)p * half + i) * 2] = cs[(size_t)i]; tab[((size_t)p * half + i) * 2 + 1] = sn[(size_t)i]; }
        }
        e->rope.alloc((int64_t)tab.size());
        KRAG_CUDA(cudaMemcpy(e->rope.p, tab.data(), sizeof(float) * tab.size(), cudaMemcpyHostToDevice));
    }
    e->gated = gated;
    // the classifier head of a cross-encoder (BertForSequenceClassification, one label): all four tensors or none
    const char* head[4] = {"pooler.dense.weight", "pooler.dense.bias", "classifier.weight", "classifier.bias"};
    const int64_t head_n[4] = {(int64_t)d * d, d, d, 1};
    int n_head = 0;
    for (int j = 0; j < 4; ++j) {
        auto it = e->t.find(head[j]);
        if (it == e->t.end() || !it->second.p) continue;
        if (it->second.cap != head_n[j])
            throw std::runtime_error(std::string("embedder: ") + head[j] + " must hold " + std::to_string(head_n[j]) + " elements");
        ++n_head;
    }
    if (n_head != 0 && n_head != 4) throw std::runtime_error("embedder: the classifier head needs pooler.dense.{weight,bias} and classifier.{weight,bias}");
    if (n_head == 4) {
        e->s_pool = emb_split_weight(e, emb_get(e, "pooler.dense.weight", (int64_t)d * d), (size_t)d * d);
        e->has_head = true;
    }
    if (e->li_dim) {
        const int pad = (e->li_dim + GM_TILE - 1) / GM_TILE * GM_TILE;
        DevArray<float> w;
        w.alloc((int64_t)pad * d);
        KRAG_CUDA(cudaMemsetAsync(w.p, 0, sizeof(float) * (size_t)pad * d, e->st));
        KRAG_CUDA(cudaMemcpyAsync(w.p, emb_get(e, LI_WEIGHT, (int64_t)e->li_dim * d), sizeof(float) * (size_t)e->li_dim * d,
                                  cudaMemcpyDeviceToDevice, e->st));
        e->s_li = emb_split_weight(e, w.p, (size_t)pad * d);
        e->li_bias.alloc(pad);
        KRAG_CUDA(cudaMemsetAsync(e->li_bias.p, 0, sizeof(float) * (size_t)pad, e->st));
        KRAG_CUDA(cudaStreamSynchronize(e->st));   // w is freed at scope end
        e->li_pad = pad;
    }
    if (rel) {
        // the bias by distance, [heads][REL_TAB]: the kernel looks a score's bias up without computing its bucket
        std::vector<float> w((size_t)REL_BUCKETS * c.heads), tab((size_t)c.heads * REL_TAB);
        KRAG_CUDA(cudaMemcpy(w.data(), emb_get(e, REL_BIAS, (int64_t)w.size()), sizeof(float) * w.size(), cudaMemcpyDeviceToHost));
        for (int h = 0; h < c.heads; ++h)
            for (int dist = -REL_MAX; dist <= REL_MAX; ++dist)
                tab[(size_t)h * REL_TAB + dist + REL_MAX] = w[(size_t)relative_bucket(dist) * c.heads + h];
        e->rel_tab.alloc((int64_t)tab.size());
        KRAG_CUDA(cudaMemcpy(e->rel_tab.p, tab.data(), sizeof(float) * tab.size(), cudaMemcpyHostToDevice));
    }
    KRAG_CUDA(cudaStreamSynchronize(e->st));
    wtmp.release();
    // the fp32 copies of the GEMM weights are not read again: free them (the split planes hold the same bytes per element)
    for (int l = 0; l < e->cfg.layers; ++l)
        for (const char* nm : {"attention.self.query.weight", "attention.self.key.weight", "attention.self.value.weight",
                               "attention.output.dense.weight", "intermediate.dense.weight", "intermediate.gate.weight", "output.dense.weight"}) {
            auto it = e->t.find(lname(l, nm));
            if (it != e->t.end()) it->second.release();
        }
    if (!e->ws.p) e->ws.alloc((int64_t)Embedder::WS_FLOATS);
    e->finalized = true;
}

void embedder_destroy(Embedder* e)
{
    if (e->n_stores) throw std::runtime_error("embedder: destroy its passage vector stores first");
    delete e;
}

int embedder_hidden(const Embedder* e) { return e->cfg.hidden; }

void embedder_set_pooling(Embedder* e, int mode)
{
    if (mode != EMB_POOL_CLS && mode != EMB_POOL_MEAN) throw std::runtime_error("embedder: pooling mode must be CLS or MEAN");
    e->pooling = mode;
}

void embedder_set_cls_rows_only(Embedder* e, bool on) { e->cls_rows_only = on; }

// The weights' hi planes ARE their fp16 values, so the two modes share one copy and the mode can change between forwards.
void embedder_set_precision(Embedder* e, int mode)
{
    if (mode != EMB_PREC_FP32 && mode != EMB_PREC_FP16) throw std::runtime_error("embedder: precision must be FP32 or FP16");
    e->precision = mode;
}

void embedder_set_position_offset(Embedder* e, int off)
{
    if (off < 0) throw std::runtime_error("embedder: the position offset must be >= 0");
    e->pos_off = off;
}

template <int G>
static void launch_mean_normalize(const float* x, const int32_t* seq_off, float* out, int batch, int ld_out, cudaStream_t st)
{
    mean_normalize_kernel<G><<<(unsigned)batch, MP_WARPS * 32, 0, st>>>(x, seq_off, out, ld_out);
}
// the final writer: pooled, L2-normalised embeddings of the residual stream x (cls_rows: of the [CLS] rows in cx) into rows
// of stride ld_out
static void launch_pool(const Embedder* e, int batch, bool cls_rows, float* out, int ld_out, cudaStream_t st)
{
    const int d = e->cfg.hidden;
    if (e->pooling == EMB_POOL_MEAN) {
        switch (d / 128) {             // embedder_create: d % 128 == 0, d <= 1024
        case 1: launch_mean_normalize<1>(e->x.p, e->d_off.p, out, batch, ld_out, st); break;
        case 2: launch_mean_normalize<2>(e->x.p, e->d_off.p, out, batch, ld_out, st); break;
        case 3: launch_mean_normalize<3>(e->x.p, e->d_off.p, out, batch, ld_out, st); break;
        case 4: launch_mean_normalize<4>(e->x.p, e->d_off.p, out, batch, ld_out, st); break;
        case 5: launch_mean_normalize<5>(e->x.p, e->d_off.p, out, batch, ld_out, st); break;
        case 6: launch_mean_normalize<6>(e->x.p, e->d_off.p, out, batch, ld_out, st); break;
        case 7: launch_mean_normalize<7>(e->x.p, e->d_off.p, out, batch, ld_out, st); break;
        default: launch_mean_normalize<8>(e->x.p, e->d_off.p, out, batch, ld_out, st); break;
        }
    } else {
        cls_normalize_kernel<<<(batch * 32 + 255) / 256, 256, 0, st>>>(cls_rows ? e->cx.p : e->x.p, cls_rows ? nullptr : e->d_off.p, out, batch,
                                                                        d, ld_out);
    }
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// The encoder over packed sequences (tok_ids, tok_offsets [batch+1], host) up to the last hidden state, enqueued on e->st.
// seg_b (host, [batch] or null): index of the first token of segment B of each sequence; tokens from there on add token
// type row 1, the others row 0 (null: row 0 everywhere, the single-sequence embedding).  cls_ok: only the [CLS] rows of the
// last layer are read.  Returns whether the last layer ran on the [CLS] rows only (then in cx / cxs, else x / xs).
// late (late-interaction token vectors): every row of the last layer is read, and each sequence's rows get bits that depend
// on its own tokens alone -- every GEMM runs the one plan LATE_PLAN (linear_plan picks the tile width and K split from the
// token count) and attention the 64-key blocking whatever the batch's longest sequence.  kv_len (host, [batch] or null; late only): the
// keys of sequence b are its first kv_len[b] rows.
constexpr GemmPlan LATE_PLAN{128, 1, false};   // 128 x 128 tiles, the whole K range: valid for every N % 128 == 0 (hidden, 3 hidden, FFN)
static bool encoder_forward(Embedder* e, int batch, const int32_t* tok_ids, const int32_t* tok_offsets, const int32_t* seg_b, bool cls_ok,
                            bool late = false, const int32_t* kv_len = nullptr)
{
    if (!e->finalized) throw std::runtime_error("embedder: call finalize after loading the weights");
    const BertConfig& c = e->cfg;
    const int d = c.hidden, n_tok = tok_offsets[batch];
    cudaStream_t st = e->st;
    int max_len = 0;
    std::vector<int32_t> pos((size_t)n_tok), typ(seg_b ? (size_t)n_tok : 0);
    if (seg_b && c.type_vocab < 2)          // finalize: the token type table holds type_vocab rows
        throw std::runtime_error("embedder: sentence pairs need token type row 1 (type_vocab_size >= 2)");
    const int off = e->pos_off;
    for (int b = 0; b < batch; ++b) {
        const int len = tok_offsets[b + 1] - tok_offsets[b];
        if (len < 1 || len > c.max_pos - off)
            throw std::runtime_error("embedder: sequence length must be in [1, max_position - position offset]");
        max_len = len > max_len ? len : max_len;
        if (kv_len && (kv_len[b] < 1 || kv_len[b] > len)) throw std::runtime_error("embedder: a key length must be in [1, sequence length]");
        for (int i = 0; i < len; ++i) pos[(size_t)tok_offsets[b] + i] = off + i;
        if (seg_b) {
            if (seg_b[b] < 1 || seg_b[b] > len) throw std::runtime_error("embedder: segment B must start in [1, sequence length]");
            for (int i = 0; i < len; ++i) typ[(size_t)tok_offsets[b] + i] = i >= seg_b[b] ? 1 : 0;
        }
    }
    if (n_tok > e->cap_tok || batch > e->cap_batch) {
        const int64_t T = n_tok > e->cap_tok ? n_tok : e->cap_tok, Bc = batch > e->cap_batch ? batch : e->cap_batch;
        e->drop_graphs(); e->seen.clear();   // captured pointers are about to change
        KRAG_CUDA(cudaStreamSynchronize(st));
        // all old buffers go before the first new one is allocated (the peak is the new set only); a grow that fails
        // half-way leaves no workspace and capacity 0, so the next call grows again
        e->cap_tok = e->cap_batch = 0;
        e->d_tok.release(); e->d_pos.release(); e->d_off.release(); e->d_typ.release(); e->d_kvl.release(); e->x.release(); e->x2.release(); e->qkv.release();
        e->xs.release(); e->cs.release(); e->fs.release(); e->out.release();
        e->cx.release(); e->cx2.release(); e->ccs.release(); e->cxs.release(); e->cfs.release();
        e->d_tok.alloc(T); e->d_pos.alloc(T); e->d_off.alloc(Bc + 1); e->d_typ.alloc(T); e->d_kvl.alloc(Bc);
        e->x.alloc(T * d); e->x2.alloc(T * d); e->qkv.alloc(2 * T * 3 * d);
        e->xs.alloc(2 * T * d); e->cs.alloc(2 * T * d); e->fs.alloc(2 * T * c.inter);
        e->out.alloc(Bc * d);
        e->cx.alloc(Bc * d); e->cx2.alloc(Bc * d); e->ccs.alloc(2 * Bc * d); e->cxs.alloc(2 * Bc * d); e->cfs.alloc(2 * Bc * c.inter);
        e->cap_tok = (int)T; e->cap_batch = (int)Bc;
    }
    // split planes: [hi plane | lo plane], each cap_tok rows.  planes == 1 (fp16 precision): no producer writes a lo plane and
    // no product reads one
    const int planes = e->precision == EMB_PREC_FP16 ? 1 : 2;
    auto lo_of = [&](uint16_t* hi, size_t n) -> uint16_t* { return planes == 2 ? hi + n : nullptr; };
    const SplitMat xs{e->xs.p, lo_of(e->xs.p, (size_t)e->cap_tok * d)}, cs{e->cs.p, lo_of(e->cs.p, (size_t)e->cap_tok * d)},
                   fs{e->fs.p, lo_of(e->fs.p, (size_t)e->cap_tok * c.inter)};
    KRAG_CUDA(cudaMemcpyAsync(e->d_tok.p, tok_ids, 4 * (size_t)n_tok, cudaMemcpyHostToDevice, st));
    KRAG_CUDA(cudaMemcpyAsync(e->d_pos.p, pos.data(), 4 * (size_t)n_tok, cudaMemcpyHostToDevice, st));
    KRAG_CUDA(cudaMemcpyAsync(e->d_off.p, tok_offsets, 4 * (size_t)(batch + 1), cudaMemcpyHostToDevice, st));
    if (seg_b) KRAG_CUDA(cudaMemcpyAsync(e->d_typ.p, typ.data(), 4 * (size_t)n_tok, cudaMemcpyHostToDevice, st));
    if (kv_len) KRAG_CUDA(cudaMemcpyAsync(e->d_kvl.p, kv_len, 4 * (size_t)batch, cudaMemcpyHostToDevice, st));
    const GemmPlan* const plan = late ? &LATE_PLAN : nullptr;
    const int att_len = late && max_len <= 64 ? 65 : max_len;   // the attention blocking of sequences over 64 tokens
    const int32_t* const d_kvl = kv_len ? e->d_kvl.p : nullptr;

    // CLS pooling reads one row per sequence of the last layer's output.  K and V of every token are still needed, so the
    // last QKV projection runs over all tokens; attention then runs for the first query rows only, and the O projection,
    // FFN and LayerNorms run on the gathered [CLS] rows.  Those GEMMs keep the plan (tile width, K split) of the full
    // token count, so every [CLS] row gets the same bits as in the full layer.  Taken when it saves a 128-row tile.
    const bool cls_rows = !late && cls_ok && e->cls_rows_only && (n_tok + GM_TILE - 1) / GM_TILE > (batch + GM_TILE - 1) / GM_TILE;
    // The forward is ~7 kernels per layer; for a handful of query tokens it is bound by launch gaps and kernel
    // prologues, so each (n_tok, batch, max_len, cls_rows, head) shape is captured into a CUDA graph the second time it is seen.
    const int dh = d / c.heads;
    // rotary encoders: no position row; Q and K are rotated in the QKV epilogue.  Gated FFN: FFN1 has 2 * inter columns
    const bool rotary = e->rope.p != nullptr;
    const EpiArgs ep_qkv{rotary ? EP_ROPE : EP_PLAIN, e->rope.p, e->d_pos.p, 2 * d, dh / 2};
    const EpiArgs ep_f1{e->gated ? EP_SWIGLU : EP_PLAIN, nullptr, nullptr, 0, 0};
    const int n_f1 = e->gated ? 2 * c.inter : c.inter;
    auto f1_bias = [&](int l) { return e->gated ? e->bf1[(size_t)l].p : e->t[lname(l, "intermediate.dense.bias")].p; };
    auto run_layers = [&]() {
    if (rotary)
        launch_pdl(embed_ln_kernel<false>, dim3((unsigned)((n_tok + 7) / 8)), dim3(256), (size_t)8 * d * 4, st, e->d_tok.p, nullptr,
                   seg_b ? e->d_typ.p : nullptr, e->t["embeddings.word_embeddings.weight"].p, nullptr,
                   e->t["embeddings.token_type_embeddings.weight"].p, e->t["embeddings.LayerNorm.weight"].p, e->t["embeddings.LayerNorm.bias"].p,
                   e->x.p, xs.hi, xs.lo, n_tok, d, c.vocab, c.eps);
    else
        launch_pdl(embed_ln_kernel<true>, dim3((unsigned)((n_tok + 7) / 8)), dim3(256), (size_t)8 * d * 4, st, e->d_tok.p, e->d_pos.p,
                   seg_b ? e->d_typ.p : nullptr, e->t["embeddings.word_embeddings.weight"].p, e->t["embeddings.position_embeddings.weight"].p,
                   e->t["embeddings.token_type_embeddings.weight"].p, e->t["embeddings.LayerNorm.weight"].p, e->t["embeddings.LayerNorm.bias"].p, e->x.p,
                   xs.hi, xs.lo, n_tok, d, c.vocab, c.eps);
    // the QKV projection writes the split planes only (same bytes as an fp32 matrix); attention reads them on the tensor cores
    uint16_t* q_hi = e->qkv.p;
    uint16_t* q_lo = lo_of(q_hi, (size_t)n_tok * 3 * d);
    for (int l = 0; l < c.layers; ++l) {
        const size_t L = (size_t)l;
        const bool last_cls = cls_rows && l == c.layers - 1;
        launch_linear(e->di, xs, e->s_qkv[L], n_tok, 3 * d, d, e->bqkv[L].p, nullptr, false, nullptr, q_hi, q_lo, nullptr, nullptr, 0.f,
                      nullptr, nullptr, nullptr, e->ws.p, Embedder::WS_FLOATS, st, plan, planes, &ep_qkv);
        const float* rel = e->rel_tab.p;                  // null: BERT
        if (planes == 1) {
            if (dh == 64) attention_mma<64, 1>(q_hi, q_lo, e->d_off.p, cs.hi, cs.lo, d, c.heads, batch, att_len, last_cls, rel, d_kvl, st);
            else attention_mma<32, 1>(q_hi, q_lo, e->d_off.p, cs.hi, cs.lo, d, c.heads, batch, att_len, last_cls, rel, d_kvl, st);
        } else if (dh == 64) attention_mma<64, 2>(q_hi, q_lo, e->d_off.p, cs.hi, cs.lo, d, c.heads, batch, att_len, last_cls, rel, d_kvl, st);
        else attention_mma<32, 2>(q_hi, q_lo, e->d_off.p, cs.hi, cs.lo, d, c.heads, batch, att_len, last_cls, rel, d_kvl, st);
        if (last_cls) {
            const SplitMat ccs{e->ccs.p, lo_of(e->ccs.p, (size_t)batch * d)}, cxs{e->cxs.p, lo_of(e->cxs.p, (size_t)batch * d)},
                           cfs{e->cfs.p, lo_of(e->cfs.p, (size_t)batch * c.inter)};
            const GemmPlan po = linear_plan(e->di, n_tok, d, d, true, true, Embedder::WS_FLOATS, planes);
            const GemmPlan p1 = linear_plan(e->di, n_tok, n_f1, d, false, true, Embedder::WS_FLOATS, planes);
            const GemmPlan p2 = linear_plan(e->di, n_tok, d, c.inter, true, true, Embedder::WS_FLOATS, planes);
            launch_pdl(gather_cls_kernel, dim3((unsigned)((batch * 32 + 255) / 256)), dim3(256), 0, st, e->x.p, cs.hi, cs.lo, e->d_off.p, e->cx.p,
                       ccs.hi, ccs.lo, batch, d);
            launch_linear(e->di, ccs, e->s_o[L], batch, d, d, e->t[lname(l, "attention.output.dense.bias")].p, e->cx.p, false, e->cx2.p, nullptr,
                          nullptr, e->t[lname(l, "attention.output.LayerNorm.weight")].p, e->t[lname(l, "attention.output.LayerNorm.bias")].p, c.eps,
                          e->cx.p, cxs.hi, cxs.lo, e->ws.p, Embedder::WS_FLOATS, st, &po, planes);
            launch_linear(e->di, cxs, e->s_f1[L], batch, n_f1, d, f1_bias(l), nullptr, !e->gated, nullptr, cfs.hi,
                          cfs.lo, nullptr, nullptr, 0.f, nullptr, nullptr, nullptr, e->ws.p, Embedder::WS_FLOATS, st, &p1, planes, &ep_f1);
            launch_linear(e->di, cfs, e->s_f2[L], batch, d, c.inter, e->t[lname(l, "output.dense.bias")].p, e->cx.p, false, e->cx2.p, nullptr,
                          nullptr, e->t[lname(l, "output.LayerNorm.weight")].p, e->t[lname(l, "output.LayerNorm.bias")].p, c.eps, e->cx.p, cxs.hi,
                          cxs.lo, e->ws.p, Embedder::WS_FLOATS, st, &p2, planes);
            break;
        }
        // O projection (+bias +residual) -> LayerNorm -> x (fp32 residual stream) + its split planes
        launch_linear(e->di, cs, e->s_o[L], n_tok, d, d, e->t[lname(l, "attention.output.dense.bias")].p, e->x.p, false, e->x2.p, nullptr, nullptr,
                      e->t[lname(l, "attention.output.LayerNorm.weight")].p, e->t[lname(l, "attention.output.LayerNorm.bias")].p, c.eps, e->x.p, xs.hi, xs.lo,
                      e->ws.p, Embedder::WS_FLOATS, st, plan, planes);
        // FFN1 (+bias, GELU; gated: silu(gate) * up): only the split planes are written (FFN2 is the sole consumer)
        launch_linear(e->di, xs, e->s_f1[L], n_tok, n_f1, d, f1_bias(l), nullptr, !e->gated, nullptr, fs.hi, fs.lo,
                      nullptr, nullptr, 0.f, nullptr, nullptr, nullptr, e->ws.p, Embedder::WS_FLOATS, st, plan, planes, &ep_f1);
        // FFN2 (+bias +residual) -> LayerNorm -> x + split planes
        launch_linear(e->di, fs, e->s_f2[L], n_tok, d, c.inter, e->t[lname(l, "output.dense.bias")].p, e->x.p, false, e->x2.p, nullptr, nullptr,
                      e->t[lname(l, "output.LayerNorm.weight")].p, e->t[lname(l, "output.LayerNorm.bias")].p, c.eps, e->x.p, xs.hi, xs.lo, e->ws.p,
                      Embedder::WS_FLOATS, st, plan, planes);
    }
    };   // run_layers
    const Embedder::GraphKey key(n_tok, batch, max_len, cls_rows ? 1 : 0, seg_b ? 1 : 0, e->precision, late ? (kv_len ? 2 : 1) : 0);
    auto git = e->graphs.find(key);
    if (git != e->graphs.end()) {
        KRAG_CUDA(cudaGraphLaunch(git->second, st));
        count_launch(1 + 7 * c.layers + (cls_rows ? 1 : 0));
    } else if (e->seen.size() > 4096 ? (e->seen.clear(), false) : e->seen[key]++ >= 1) {
        if (e->graphs.size() >= 64) e->drop_graphs();
        cudaGraph_t g = nullptr;
        cudaGraphExec_t ex = nullptr;
        KRAG_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        try { run_layers(); } catch (...) { cudaStreamEndCapture(st, &g); if (g) cudaGraphDestroy(g); throw; }
        KRAG_CUDA(cudaStreamEndCapture(st, &g));
        KRAG_CUDA(cudaGraphInstantiate(&ex, g, 0));
        KRAG_CUDA(cudaGraphDestroy(g));
        e->graphs[key] = ex;
        KRAG_CUDA(cudaGraphLaunch(ex, st));
    } else {
        run_layers();
    }
    return cls_rows;
}

// tok_ids: packed tokens of all sequences; tok_offsets [batch+1]; out_host [batch, hidden]
// out_host != nullptr: embeddings are copied to the host and the call returns synchronised.
// out_dev  != nullptr: embeddings are written to device rows of stride ld_out floats and `consumer` (a stream of
//                      the caller) is made to wait for them -- no host round trip.
void embedder_forward(Embedder* e, int batch, const int32_t* tok_ids, const int32_t* tok_offsets, float* out_host,
                      float* out_dev, int ld_out, cudaStream_t consumer)
{
    const bool cls_rows = encoder_forward(e, batch, tok_ids, tok_offsets, nullptr, e->pooling == EMB_POOL_CLS);
    const int d = e->cfg.hidden;
    cudaStream_t st = e->st;
    if (out_dev) {
        // the caller's buffer may still be read by work it enqueued earlier on `consumer` (the previous batch's scan): only
        // the final writer waits for that; the forward itself overlaps with it
        if (!e->in_ev) KRAG_CUDA(cudaEventCreateWithFlags(&e->in_ev, cudaEventDisableTiming));
        KRAG_CUDA(cudaEventRecord(e->in_ev, consumer));
        KRAG_CUDA(cudaStreamWaitEvent(st, e->in_ev, 0));
        launch_pool(e, batch, cls_rows, out_dev, ld_out, st);
        if (!e->done) KRAG_CUDA(cudaEventCreateWithFlags(&e->done, cudaEventDisableTiming));
        KRAG_CUDA(cudaEventRecord(e->done, st));
        KRAG_CUDA(cudaStreamWaitEvent(consumer, e->done, 0));
    }
    if (out_host) {
        launch_pool(e, batch, cls_rows, e->out.p, d, st);
        KRAG_CUDA(cudaMemcpyAsync(out_host, e->out.p, 4 * (size_t)batch * d, cudaMemcpyDeviceToHost, st));
        KRAG_CUDA(cudaStreamSynchronize(st));
    }
}

// Cross-encoder reranking.  Pairs [CLS] q [SEP] d [SEP] of n_queries queries, packed: query i owns pairs
// pair_off[i] .. pair_off[i + 1] (at most RERANK_MAX_CANDIDATES), pair p is tok_ids[tok_off[p] .. tok_off[p + 1]) with
// segment B from seg_b[p]; seg_b null (XLM-R's <s> q </s></s> d </s>): type row 0 for every token.  The pairs go through forwards of at most RERANK_MAX_TOKENS tokens (whole pairs), each followed by
// the pooler GEMM and the classifier head, which write the pair's score at its offset in one buffer; one select kernel then
// orders every query's scores and one copy brings back [n_queries, top_k] positions (within the query's pairs, -1 past its
// count) and scores.
void embedder_rerank(Embedder* e, int n_queries, const int32_t* pair_off, const int32_t* tok_ids, const int32_t* tok_off,
                     const int32_t* seg_b, int act, int top_k, int32_t* out_pos, float* out_score)
{
    if (!e->finalized) throw std::runtime_error("embedder: call finalize after loading the weights");
    if (!e->has_head) throw std::runtime_error("embedder: reranking needs the classifier head (pooler.dense.*, classifier.*)");
    if (act != EMB_ACT_SIGMOID && act != EMB_ACT_IDENTITY) throw std::runtime_error("embedder: unknown head activation");
    if (top_k < 1 || top_k > RERANK_MAX_CANDIDATES) throw std::runtime_error("embedder: top_k must be in [1, 300]");
    if (n_queries < 1 || pair_off[0] != 0) throw std::runtime_error("embedder: pair offsets must start at 0");
    for (int q = 0; q < n_queries; ++q) {
        const int n = pair_off[q + 1] - pair_off[q];
        if (n < 0 || n > RERANK_MAX_CANDIDATES) throw std::runtime_error("embedder: a query has 0 to 300 candidate pairs");
    }
    const int n_pairs = pair_off[n_queries], d = e->cfg.hidden;
    if (n_pairs > 0 && tok_off[0] != 0) throw std::runtime_error("embedder: token offsets must start at 0");
    for (int p = 0; p < n_pairs; ++p) {
        const int len = tok_off[p + 1] - tok_off[p];
        if (len < 1 || len > e->cfg.max_pos - e->pos_off)
            throw std::runtime_error("embedder: a pair's length must be in [1, max_position - position offset]");
    }
    cudaStream_t st = e->st;
    if (e->scores.cap < (n_pairs > 0 ? n_pairs : 1)) e->scores.alloc(n_pairs > 0 ? n_pairs : 1);
    if (e->d_poff.cap < n_queries + 1) e->d_poff.alloc(n_queries + 1);
    if (e->sel.cap < 2 * (int64_t)n_queries * top_k) e->sel.alloc(2 * (int64_t)n_queries * top_k);
    std::vector<int32_t> offs;
    for (int p0 = 0; p0 < n_pairs;) {
        int p1 = p0 + 1;
        while (p1 < n_pairs && tok_off[p1 + 1] - tok_off[p0] <= RERANK_MAX_TOKENS) ++p1;
        const int batch = p1 - p0;
        offs.assign((size_t)batch + 1, 0);
        for (int j = 0; j <= batch; ++j) offs[(size_t)j] = tok_off[p0 + j] - tok_off[p0];
        const bool cls_rows = encoder_forward(e, batch, tok_ids + tok_off[p0], offs.data(), seg_b ? seg_b + p0 : nullptr, true);
        // the [CLS] rows' split planes: where the shortened last layer left them, else gathered from the full stream
        const int planes = e->precision == EMB_PREC_FP16 ? 1 : 2;
        const SplitMat cxs{e->cxs.p, planes == 2 ? e->cxs.p + (size_t)batch * d : nullptr};
        if (!cls_rows) {
            const SplitMat xs{e->xs.p, planes == 2 ? e->xs.p + (size_t)e->cap_tok * d : nullptr};
            launch_pdl(gather_cls_kernel, dim3((unsigned)((batch * 32 + 255) / 256)), dim3(256), 0, st, e->x.p, xs.hi, xs.lo, e->d_off.p,
                       e->cx.p, cxs.hi, cxs.lo, batch, d);
        }
        launch_linear(e->di, cxs, e->s_pool, batch, d, d, e->t["pooler.dense.bias"].p, nullptr, false, e->cx2.p, nullptr, nullptr, nullptr,
                      nullptr, 0.f, nullptr, nullptr, nullptr, e->ws.p, Embedder::WS_FLOATS, st, nullptr, planes);
        classifier_head_kernel<<<(unsigned)((batch * 32 + 255) / 256), 256, 0, st>>>(e->cx2.p, e->t["classifier.weight"].p,
                                                                                   e->t["classifier.bias"].p, batch, d, act, e->scores.p + p0);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        p0 = p1;
    }
    KRAG_CUDA(cudaMemcpyAsync(e->d_poff.p, pair_off, 4 * (size_t)(n_queries + 1), cudaMemcpyHostToDevice, st));
    const size_t nk = (size_t)n_queries * top_k;
    rerank_select_kernel<<<(unsigned)n_queries, 256, 0, st>>>(e->scores.p, e->d_poff.p, top_k, e->sel.p,
                                                             reinterpret_cast<float*>(e->sel.p + nk));
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    std::vector<int32_t> h(2 * nk);
    KRAG_CUDA(cudaMemcpyAsync(h.data(), e->sel.p, 4 * 2 * nk, cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    std::memcpy(out_pos, h.data(), 4 * nk);
    std::memcpy(out_score, h.data() + nk, 4 * nk);
}


// ---- late interaction (ColBERT)
// Unit token vectors of packed sequences: the late-interaction forward (every row of the last layer, bits per sequence),
// the projection W . h through the split-fp16 GEMM with zero bias into [n_tok][li_pad] (columns past li_dim are exact zeros),
// then cls_normalize_kernel over every row (one warp per row, fixed fp32 order; the zero columns add nothing to the norm),
// written to rows of `out` (device, stride li_pad).  Sequences go through forwards of at most RERANK_MAX_TOKENS tokens.
static void late_vectors(Embedder* e, int batch, const int32_t* tok_ids, const int32_t* tok_off, const int32_t* kv_len, float* out)
{
    const int d = e->cfg.hidden, pad = e->li_pad;
    const int planes = e->precision == EMB_PREC_FP16 ? 1 : 2;
    std::vector<int32_t> offs;
    for (int b0 = 0; b0 < batch;) {
        int b1 = b0 + 1;
        while (b1 < batch && tok_off[b1 + 1] - tok_off[b0] <= RERANK_MAX_TOKENS) ++b1;
        const int nb = b1 - b0, n_tok = tok_off[b1] - tok_off[b0];
        offs.assign((size_t)nb + 1, 0);
        for (int j = 0; j <= nb; ++j) offs[(size_t)j] = tok_off[b0 + j] - tok_off[b0];
        encoder_forward(e, nb, tok_ids + tok_off[b0], offs.data(), nullptr, false, true, kv_len ? kv_len + b0 : nullptr);
        if (e->li_c.cap < (int64_t)e->cap_tok * pad) e->li_c.alloc((int64_t)e->cap_tok * pad);
        const SplitMat xs{e->xs.p, planes == 2 ? e->xs.p + (size_t)e->cap_tok * d : nullptr};
        launch_linear(e->di, xs, e->s_li, n_tok, pad, d, e->li_bias.p, nullptr, false, e->li_c.p, nullptr, nullptr, nullptr, nullptr, 0.f,
                      nullptr, nullptr, nullptr, nullptr, 0, e->st, &LATE_PLAN, planes);
        cls_normalize_kernel<<<(unsigned)((n_tok * 32 + 255) / 256), 256, 0, e->st>>>(e->li_c.p, nullptr, out + (size_t)tok_off[b0] * pad,
                                                                                     n_tok, pad, pad);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
        b0 = b1;
    }
}

static void late_check(const Embedder* e, int batch, const int32_t* tok_off)
{
    if (!e->finalized) throw std::runtime_error("embedder: call finalize after loading the weights");
    if (!e->li_pad) throw std::runtime_error("embedder: late interaction needs krag_embedder_set_late_interaction before finalize");
    if (batch < 1 || tok_off[0] != 0) throw std::runtime_error("embedder: token offsets must start at 0");
    for (int b = 0; b < batch; ++b) {
        const int len = tok_off[b + 1] - tok_off[b];
        if (len < 1 || len > e->cfg.max_pos - e->pos_off)
            throw std::runtime_error("embedder: sequence length must be in [1, max_position - position offset]");
    }
}

void embedder_late_vectors(Embedder* e, int batch, const int32_t* tok_ids, const int32_t* tok_off, const int32_t* kv_len, float* out_host)
{
    late_check(e, batch, tok_off);
    const int64_t n_tok = tok_off[batch];
    if (e->li_q.cap < n_tok * e->li_pad) e->li_q.alloc(n_tok * e->li_pad);
    late_vectors(e, batch, tok_ids, tok_off, kv_len, e->li_q.p);
    KRAG_CUDA(cudaMemcpy2DAsync(out_host, sizeof(float) * (size_t)e->li_dim, e->li_q.p, sizeof(float) * (size_t)e->li_pad,
                                sizeof(float) * (size_t)e->li_dim, (size_t)n_tok, cudaMemcpyDeviceToHost, e->st));
    KRAG_CUDA(cudaStreamSynchronize(e->st));
}

static void late_gather(Embedder* e, const float* in, const std::vector<int32_t>& src, const std::vector<float*>& dst)
{
    const int64_t n = (int64_t)src.size();
    if (n == 0) return;
    if (e->li_src.cap < n) e->li_src.alloc(n);
    if (e->li_dst.cap < n) e->li_dst.alloc(n);
    KRAG_CUDA(cudaMemcpyAsync(e->li_src.p, src.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, e->st));
    KRAG_CUDA(cudaMemcpyAsync(e->li_dst.p, dst.data(), sizeof(float*) * (size_t)n, cudaMemcpyHostToDevice, e->st));
    late_gather_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, e->st>>>(in, e->li_pad, e->li_src.p, e->li_dst.p, (int)n, e->li_dim);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

static int kept_rows(const int32_t* p_off, const uint8_t* p_keep, int p)
{
    int kept = 0;
    for (int t = p_off[p]; t < p_off[p + 1]; ++t) kept += p_keep[t] != 0;
    return kept;
}
static void check_passages(const Embedder* e, int n_pass, const int32_t* p_off, const uint8_t* p_keep)
{
    late_check(e, n_pass, p_off);
    for (int p = 0; p < n_pass; ++p)
        if (!kept_rows(p_off, p_keep, p)) throw std::runtime_error("embedder: every passage needs at least one row that enters the max");
}

// ---- passage vector stores
// A LateStore holds the kept rows of passages, per ordinal, in fixed-size device slabs (skiplist rows never enter the max,
// so they are not stored): passage o is tab[o].rows unit vectors of dim floats, contiguous from float offset tab[o].off of
// slab tab[o].slab (-1: not stored).  Passages fill the last slab in ordinal order; one that does not fit there opens a new
// slab of min(LATE_SLAB_BYTES, what the embedder's budget has left) bytes, or stays unstored when that is too small (it is
// then encoded per call).  A passage never straddles two slabs and a slab never moves, so growing the store copies nothing.
// Positions grow with the ordinal (next fit), which compaction relies on.
constexpr int64_t LATE_SLAB_BYTES = (int64_t)256 << 20;
struct LateStore {
    struct Slab { DevArray<float> a; int64_t used = 0; };
    struct Entry { int32_t slab, rows; int64_t off; };
    Embedder* e = nullptr;
    int precision = EMB_PREC_FP32, dim = 0;
    std::vector<Slab> slabs;
    std::vector<Entry> tab;
};

void embedder_set_store_budget(Embedder* e, int64_t bytes)
{
    if (bytes < 0) throw std::runtime_error("embedder: the store budget must be >= 0 bytes");
    e->store_budget = bytes;
}

LateStore* late_store_create(Embedder* e)
{
    if (!e->finalized || !e->li_pad) throw std::runtime_error("embedder: a passage vector store needs a finalized late-interaction embedder");
    LateStore* s = new LateStore;
    s->e = e; s->precision = e->precision; s->dim = e->li_dim;
    ++e->n_stores;
    return s;
}

static void store_pop_slab(LateStore* s)
{
    s->e->store_bytes -= s->slabs.back().a.bytes();
    s->slabs.pop_back();
}

void late_store_destroy(LateStore* s)
{
    while (!s->slabs.empty()) store_pop_slab(s);
    --s->e->n_stores;
    delete s;
}

static void store_check(const LateStore* s, const Embedder* e)
{
    if (s->e != e) throw std::runtime_error("embedder: the store belongs to another embedder");
    if (s->precision != e->precision) throw std::runtime_error("embedder: the store holds vectors of another precision mode");
}

// room for `rows` rows in the last slab or a new one; false: the budget (or the device) has no room
static bool store_place(LateStore* s, int rows, LateStore::Entry& en)
{
    const int64_t need = (int64_t)rows * s->dim;
    if (s->slabs.empty() || s->slabs.back().a.cap - s->slabs.back().used < need) {
        const int64_t room = std::min(LATE_SLAB_BYTES, s->e->store_budget - s->e->store_bytes) / (int64_t)sizeof(float);
        if (room < need) return false;
        LateStore::Slab sl;
        try {
            sl.a.alloc(room);
        } catch (const DevOom&) {
            return false;
        }
        s->e->store_bytes += sl.a.bytes();
        s->slabs.push_back(std::move(sl));
    }
    LateStore::Slab& sl = s->slabs.back();
    en.slab = (int32_t)s->slabs.size() - 1;
    en.off = sl.used;
    sl.used += need;
    return true;
}

// slabs past the last stored passage are freed; the last one's fill ends after that passage
static void store_trim(LateStore* s)
{
    int last = -1;
    int64_t end = 0;
    for (auto it = s->tab.rbegin(); it != s->tab.rend(); ++it)
        if (it->slab >= 0) { last = it->slab; end = it->off + (int64_t)it->rows * s->dim; break; }
    while ((int)s->slabs.size() > last + 1) store_pop_slab(s);
    if (last >= 0) s->slabs[(size_t)last].used = end;
}

// Passages p < n (tok packed by off, keep: rows that enter the max) become ordinals tab.size() + p; each is stored while
// the budget allows (stored_out[p] = 1).  Forwards follow late_vectors' RERANK_MAX_TOKENS split, and a batch without a
// stored passage runs none; late_gather_kernel copies each stored passage's kept rows into its slab, in row order.
void late_store_append(LateStore* s, int n, const int32_t* tok, const int32_t* off, const uint8_t* keep, uint8_t* stored_out)
{
    Embedder* e = s->e;
    store_check(s, e);
    check_passages(e, n, off, keep);
    const size_t n0 = s->tab.size();
    try {
        std::vector<int32_t> src, loff;
        std::vector<float*> dst;
        for (int b0 = 0; b0 < n;) {
            int b1 = b0 + 1;
            while (b1 < n && off[b1 + 1] - off[b0] <= RERANK_MAX_TOKENS) ++b1;
            src.clear(); dst.clear();
            for (int p = b0; p < b1; ++p) {
                LateStore::Entry en{-1, kept_rows(off, keep, p), 0};
                if (store_place(s, en.rows, en)) {
                    float* base = s->slabs[(size_t)en.slab].a.p + en.off;
                    int r = 0;
                    for (int t = off[p]; t < off[p + 1]; ++t)
                        if (keep[t]) { src.push_back(t - off[b0]); dst.push_back(base + (size_t)r++ * s->dim); }
                }
                s->tab.push_back(en);
                stored_out[p] = en.slab >= 0;
            }
            if (!src.empty()) {
                const int64_t n_tok = off[b1] - off[b0];
                loff.resize((size_t)(b1 - b0) + 1);
                for (int j = 0; j <= b1 - b0; ++j) loff[(size_t)j] = off[b0 + j] - off[b0];
                if (e->li_p.cap < n_tok * e->li_pad) e->li_p.alloc(n_tok * e->li_pad);
                late_vectors(e, b1 - b0, tok + off[b0], loff.data(), nullptr, e->li_p.p);
                late_gather(e, e->li_p.p, src, dst);
            }
            b0 = b1;
        }
        KRAG_CUDA(cudaStreamSynchronize(e->st));
    } catch (...) {
        s->tab.resize(n0);
        store_trim(s);
        throw;
    }
}

void late_store_truncate(LateStore* s, int64_t n)
{
    if (n < 0 || n > (int64_t)s->tab.size()) throw std::runtime_error("embedder: truncate to at most the store's ordinal count");
    s->tab.resize((size_t)n);
    store_trim(s);
}

// Keeps the ordinals whose bit is set in alive (bit o % 32 of word o / 32), renumbered 0 .. n_live - 1 in order, and moves
// their stored rows down in the same order by next fit over the same slabs: a passage goes to the first slab, from the write
// position on, with room for it.  Slabs differ in size (one opened when the budget was nearly spent is small), so that may
// skip a slab; the passage's own slab always has room at or before its old offset, so no passage moves up and the moves run
// front to back.  A move within a slab that overlaps its own source goes through a scratch buffer.  Slabs left without a
// passage are freed.  A CUDA error part way leaves rows moved under the old table: the store is then unusable (the service
// destroys it and reranks the index per call).
void late_store_compact(LateStore* s, const uint32_t* alive, int64_t n)
{
    if (n != (int64_t)s->tab.size()) throw std::runtime_error("embedder: the alive bitmap must cover every ordinal of the store");
    cudaStream_t st = s->e->st;
    std::vector<LateStore::Entry> nt;
    DevArray<float> bounce;
    int ws = 0;
    int64_t wo = 0;
    for (int64_t o = 0; o < n; ++o) {
        if (!((alive[o >> 5] >> (o & 31)) & 1u)) continue;
        LateStore::Entry en = s->tab[(size_t)o];
        if (en.slab >= 0) {
            const int64_t need = (int64_t)en.rows * s->dim;
            while (s->slabs[(size_t)ws].a.cap - wo < need) { ++ws; wo = 0; }   // stops at en.slab at the latest
            float* to = s->slabs[(size_t)ws].a.p + wo;
            const float* from = s->slabs[(size_t)en.slab].a.p + en.off;
            if (to != from) {
                const size_t bytes = sizeof(float) * (size_t)need;
                if (ws == en.slab && en.off - wo < need) {           // overlapping: source -> scratch -> destination
                    if (bounce.cap < need) {
                        KRAG_CUDA(cudaStreamSynchronize(st));       // the previous scratch's copies are done before it goes
                        bounce.alloc(need);
                    }
                    KRAG_CUDA(cudaMemcpyAsync(bounce.p, from, bytes, cudaMemcpyDeviceToDevice, st));
                    KRAG_CUDA(cudaMemcpyAsync(to, bounce.p, bytes, cudaMemcpyDeviceToDevice, st));
                } else {
                    KRAG_CUDA(cudaMemcpyAsync(to, from, bytes, cudaMemcpyDeviceToDevice, st));
                }
            }
            en.slab = ws; en.off = wo;
            wo += need;
        }
        nt.push_back(en);
    }
    KRAG_CUDA(cudaStreamSynchronize(st));
    std::vector<int32_t> keep_slab(s->slabs.size(), -1);
    for (const auto& en : nt)
        if (en.slab >= 0) keep_slab[(size_t)en.slab] = 0;
    std::vector<LateStore::Slab> kept;
    for (size_t k = 0; k < s->slabs.size(); ++k) {
        if (keep_slab[k] < 0) {
            s->e->store_bytes -= s->slabs[k].a.bytes();
            continue;                                               // freed when s->slabs is replaced below
        }
        keep_slab[k] = (int32_t)kept.size();
        kept.push_back(std::move(s->slabs[k]));
    }
    for (auto& en : nt)
        if (en.slab >= 0) en.slab = keep_slab[(size_t)en.slab];
    s->slabs = std::move(kept);
    s->tab = std::move(nt);
    store_trim(s);
}

void late_store_stats(const LateStore* s, int64_t* ordinals, int64_t* stored, int64_t* rows, int64_t* bytes)
{
    int64_t k = 0, r = 0, b = 0;
    for (const auto& en : s->tab)
        if (en.slab >= 0) { ++k; r += en.rows; }
    for (const auto& sl : s->slabs) b += sl.a.bytes();
    *ordinals = (int64_t)s->tab.size(); *stored = k; *rows = r; *bytes = b;
}

void late_store_vectors(const LateStore* s, int64_t ordinal, float* out_host, int64_t n_rows)
{
    if (ordinal < 0 || ordinal >= (int64_t)s->tab.size() || s->tab[(size_t)ordinal].slab < 0)
        throw std::runtime_error("embedder: the store does not hold ordinal " + std::to_string(ordinal));
    const LateStore::Entry& en = s->tab[(size_t)ordinal];
    if (n_rows != en.rows) throw std::runtime_error("embedder: the ordinal holds " + std::to_string(en.rows) + " rows");
    KRAG_CUDA(cudaMemcpyAsync(out_host, s->slabs[(size_t)en.slab].a.p + en.off, sizeof(float) * (size_t)n_rows * s->dim,
                              cudaMemcpyDeviceToHost, s->e->st));
    KRAG_CUDA(cudaStreamSynchronize(s->e->st));
}

// Late-interaction reranking.  n_queries queries of q_rows tokens each (q_tok [n_queries * q_rows], keys q_kv[i] <= q_rows),
// n_pass passages of the call (p_tok packed by p_off [n_pass + 1], p_keep[t] = 1 where row t enters the max), query i owns
// pairs pair_off[i] .. pair_off[i + 1].  Without a store, pair p scores passage pair_src[p] of the call; with one, pair_src[p]
// >= 0 names a stored ordinal and < 0 passage ~pair_src[p] of the call.  Each query and each passage of the call is encoded
// once and its kept rows gathered into li_k; maxsim_kernel writes every pair's score at its offset from the pair table, and
// rerank_select_kernel orders each query's scores as for krag_rerank.
static void late_rerank(Embedder* e, const LateStore* s, int n_queries, int q_rows, const int32_t* q_tok, const int32_t* q_kv, int n_pass,
                        const int32_t* p_tok, const int32_t* p_off, const uint8_t* p_keep, const int32_t* pair_off, const int32_t* pair_src,
                        int top_k, int32_t* out_pos, float* out_score)
{
    if (s) store_check(s, e);
    if (q_rows < 1 || q_rows > MS_QROWS) throw std::runtime_error("embedder: a late-interaction query holds 1 to 32 tokens");
    if (top_k < 1 || top_k > RERANK_MAX_CANDIDATES) throw std::runtime_error("embedder: top_k must be in [1, 300]");
    if (n_queries < 1 || pair_off[0] != 0) throw std::runtime_error("embedder: pair offsets must start at 0");
    for (int q = 0; q < n_queries; ++q) {
        const int n = pair_off[q + 1] - pair_off[q];
        if (n < 0 || n > RERANK_MAX_CANDIDATES) throw std::runtime_error("embedder: a query has 0 to 300 candidate pairs");
    }
    const int n_pairs = pair_off[n_queries];
    std::vector<int32_t> q_off((size_t)n_queries + 1);
    for (int q = 0; q <= n_queries; ++q) q_off[(size_t)q] = q * q_rows;
    late_check(e, n_queries, q_off.data());
    if (n_pairs == 0) n_pass = 0;
    if (n_pairs > 0 && !s && n_pass < 1) throw std::runtime_error("embedder: pairs need passages");
    if (n_pass < 0) throw std::runtime_error("embedder: the passage count must be >= 0");
    if (n_pass > 0) check_passages(e, n_pass, p_off, p_keep);
    for (int p = 0; p < n_pairs; ++p) {
        const int32_t x = pair_src[p];
        if (!s || x < 0) {
            const int32_t c = s ? ~x : x;
            if (c < 0 || c >= n_pass) throw std::runtime_error("embedder: a pair's passage index is out of range");
        } else if (x >= (int64_t)s->tab.size() || s->tab[(size_t)x].slab < 0) {
            throw std::runtime_error("embedder: a pair names ordinal " + std::to_string(x) + ", which the store does not hold");
        }
    }
    cudaStream_t st = e->st;
    const int64_t pad = e->li_pad, dim = e->li_dim, nq_tok = (int64_t)n_queries * q_rows;
    if (e->li_q.cap < nq_tok * pad) e->li_q.alloc(nq_tok * pad);
    if (e->scores.cap < (n_pairs > 0 ? n_pairs : 1)) e->scores.alloc(n_pairs > 0 ? n_pairs : 1);
    if (e->d_poff.cap < n_queries + 1) e->d_poff.alloc(n_queries + 1);
    if (e->sel.cap < 2 * (int64_t)n_queries * top_k) e->sel.alloc(2 * (int64_t)n_queries * top_k);
    late_vectors(e, n_queries, q_tok, q_off.data(), q_kv, e->li_q.p);
    KRAG_CUDA(cudaMemcpyAsync(e->d_poff.p, pair_off, 4 * (size_t)(n_queries + 1), cudaMemcpyHostToDevice, st));
    if (n_pairs > 0) {
        std::vector<int64_t> koff((size_t)n_pass + 1, 0);        // kept rows of the call's passages, packed in li_k
        if (n_pass > 0) {
            const int64_t np_tok = p_off[n_pass];
            for (int p = 0; p < n_pass; ++p) koff[(size_t)p + 1] = koff[(size_t)p] + kept_rows(p_off, p_keep, p);
            if (e->li_p.cap < np_tok * pad) e->li_p.alloc(np_tok * pad);
            if (e->li_k.cap < koff[(size_t)n_pass] * dim) e->li_k.alloc(koff[(size_t)n_pass] * dim);
            late_vectors(e, n_pass, p_tok, p_off, nullptr, e->li_p.p);
            std::vector<int32_t> src;
            std::vector<float*> dst;
            src.reserve((size_t)koff[(size_t)n_pass]); dst.reserve((size_t)koff[(size_t)n_pass]);
            for (int t = 0; t < np_tok; ++t)
                if (p_keep[t]) { dst.push_back(e->li_k.p + (size_t)src.size() * dim); src.push_back(t); }
            late_gather(e, e->li_p.p, src, dst);
        }
        std::vector<MsPair> tab((size_t)n_pairs);
        for (int p = 0; p < n_pairs; ++p) {
            const int32_t x = pair_src[p];
            if (!s || x < 0) {
                const int32_t c = s ? ~x : x;
                tab[(size_t)p] = MsPair{e->li_k.p + koff[(size_t)c] * dim, (int32_t)(koff[(size_t)c + 1] - koff[(size_t)c]), 0};
            } else {
                const LateStore::Entry& en = s->tab[(size_t)x];
                tab[(size_t)p] = MsPair{s->slabs[(size_t)en.slab].a.p + en.off, en.rows, 0};
            }
        }
        if (e->li_tab.cap < n_pairs) e->li_tab.alloc(n_pairs);
        KRAG_CUDA(cudaMemcpyAsync(e->li_tab.p, tab.data(), sizeof(MsPair) * (size_t)n_pairs, cudaMemcpyHostToDevice, st));
        int max_pairs = 0;
        for (int q = 0; q < n_queries; ++q) max_pairs = std::max(max_pairs, pair_off[q + 1] - pair_off[q]);
        const size_t smem = maxsim_smem(e->li_dim);
        static bool attr = false;
        if (!attr) { KRAG_CUDA(cudaFuncSetAttribute(maxsim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)maxsim_smem(256))); attr = true; }
        // slices per query: about four resident waves of CTAs over the call, so the last wave's tail is short
        int per_sm = 1;
        KRAG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, maxsim_kernel, MS_THREADS, smem));
        const int resident = std::max(1, per_sm) * e->di.sm_count;
        const int want = (4 * resident + n_queries - 1) / n_queries;
        const int slices = std::max(1, std::min(max_pairs, want));
        maxsim_kernel<<<dim3((unsigned)n_queries, (unsigned)slices), MS_THREADS, smem, st>>>(e->li_q.p, q_rows, (int)pad, e->li_tab.p, e->d_poff.p,
                                                                                         e->li_dim, e->scores.p);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
    }
    const size_t nk = (size_t)n_queries * top_k;
    rerank_select_kernel<<<(unsigned)n_queries, 256, 0, st>>>(e->scores.p, e->d_poff.p, top_k, e->sel.p, reinterpret_cast<float*>(e->sel.p + nk));
    KRAG_CUDA(cudaGetLastError());
    count_launch();
    std::vector<int32_t> h(2 * nk);
    KRAG_CUDA(cudaMemcpyAsync(h.data(), e->sel.p, 4 * 2 * nk, cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    std::memcpy(out_pos, h.data(), 4 * nk);
    std::memcpy(out_score, h.data() + nk, 4 * nk);
}

void embedder_late_rerank(Embedder* e, int n_queries, int q_rows, const int32_t* q_tok, const int32_t* q_kv, int n_pass, const int32_t* p_tok,
                          const int32_t* p_off, const uint8_t* p_keep, const int32_t* pair_off, const int32_t* pair_pass, int top_k,
                          int32_t* out_pos, float* out_score)
{
    late_rerank(e, nullptr, n_queries, q_rows, q_tok, q_kv, n_pass, p_tok, p_off, p_keep, pair_off, pair_pass, top_k, out_pos, out_score);
}

void late_store_rerank(Embedder* e, const LateStore* s, int n_queries, int q_rows, const int32_t* q_tok, const int32_t* q_kv, int n_pass,
                       const int32_t* p_tok, const int32_t* p_off, const uint8_t* p_keep, const int32_t* pair_off, const int32_t* pair_src,
                       int top_k, int32_t* out_pos, float* out_score)
{
    late_rerank(e, s, n_queries, q_rows, q_tok, q_kv, n_pass, p_tok, p_off, p_keep, pair_off, pair_src, top_k, out_pos, out_score);
}

}  // namespace krag
