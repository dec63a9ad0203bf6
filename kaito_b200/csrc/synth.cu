// synth.cu -- deterministic synthetic corpora generated on the device (bench / full-size
// property tests only; not on the product path).  SURVEY.md section 8(d):
//   dense : x = normalize(N(0,1)^d), Philox4x32-10, key = seed, counter = (row, block)
//   sparse: doc length ~ clip(lognormal(ln 96, 0.6), 8, 512); terms ~ power law s = 1.07
//           over [0, vocab) (continuous inverse-CDF Zipf); tf = multiplicity
#include <cub/device/device_scan.cuh>

#include "engine.h"
#include "common.cuh"

namespace krag {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k)
{
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
        uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += W0; k.y += W1;
    }
    return c;
}
__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }  // (0,1)

// one warp per row
__global__ void __launch_bounds__(256)
synth_dense_kernel(float* __restrict__ X, int64_t n, int d, int dpad, int64_t row_base, uint64_t seed)
{
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n) return;
    const uint64_t g = (uint64_t)(row_base + r);
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ 0x4B414954u);  // "KAIT"
    float* row = X + r * dpad;
    float ss = 0.f;
    for (int i0 = lane * 4; i0 < dpad; i0 += 128) {
        uint4 rnd = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), (uint32_t)(i0 >> 2), 0u), key);
        float r0 = sqrtf(-2.f * __logf(u01(rnd.x))), r1 = sqrtf(-2.f * __logf(u01(rnd.z)));
        float s0, c0, s1, c1;
        __sincosf(6.2831853f * u01(rnd.y), &s0, &c0);
        __sincosf(6.2831853f * u01(rnd.w), &s1, &c1);
        float4 v = make_float4(r0 * c0, r0 * s0, r1 * c1, r1 * s1);
        if (i0 + 0 >= d) v.x = 0.f;
        if (i0 + 1 >= d) v.y = 0.f;
        if (i0 + 2 >= d) v.z = 0.f;
        if (i0 + 3 >= d) v.w = 0.f;
        ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
        *reinterpret_cast<float4*>(row + i0) = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float inv = rsqrtf(ss);
    __syncwarp();
    for (int i0 = lane * 4; i0 < dpad; i0 += 128) {
        float4 v = *reinterpret_cast<float4*>(row + i0);
        v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
        *reinterpret_cast<float4*>(row + i0) = v;
    }
}

void launch_synth_dense(float* X, int64_t n, int d, int dpad, int64_t row_base, uint64_t seed, cudaStream_t st)
{
    if (n == 0) return;
    int64_t threads = n * 32;
    synth_dense_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(X, n, d, dpad, row_base, seed);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// ------------------------------------------------------------------------------ sparse
constexpr int SY_MAX_LEN = 512;
constexpr int SY_WARPS = 8;

__device__ __forceinline__ int synth_doc_len(uint64_t g, uint2 key)
{
    uint4 rnd = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), 0xFFFFFFFFu, 1u), key);
    float z = sqrtf(-2.f * __logf(u01(rnd.x))) * __cosf(6.2831853f * u01(rnd.y));
    float len = __expf(4.5643482f /* ln 96 */ + 0.6f * z);
    int dl = (int)len;
    return dl < 8 ? 8 : (dl > SY_MAX_LEN ? SY_MAX_LEN : dl);
}
__device__ __forceinline__ uint32_t synth_term(float u, float vmax_pow, float inv_exp, int64_t vocab)
{
    // continuous power law on [1, vocab+1): x = (1 + u * ((V+1)^(1-s) - 1))^(1/(1-s))
    float x = __powf(1.f + u * (vmax_pow - 1.f), inv_exp);
    int64_t t = (int64_t)x - 1;
    return (uint32_t)(t < 0 ? 0 : (t >= vocab ? vocab - 1 : t));
}

// mode 0: count unique terms per doc (uniq[d], doc_len[d]); mode 1: write term ids / tf at offsets
template <int MODE>
__global__ void __launch_bounds__(SY_WARPS * 32)
synth_sparse_kernel(int64_t n, int64_t row_base, uint64_t seed, int64_t vocab, float vmax_pow, float inv_exp,
                    int64_t* __restrict__ uniq, uint32_t* __restrict__ doc_len, const int64_t* __restrict__ offsets,
                    uint32_t* __restrict__ term_ids, uint16_t* __restrict__ term_tf)
{
    __shared__ uint32_t s_tok[SY_WARPS][SY_MAX_LEN];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t d = (int64_t)blockIdx.x * SY_WARPS + warp;
    if (d >= n) return;
    const uint64_t g = (uint64_t)(row_base + d);
    const uint2 key = make_uint2((uint32_t)seed ^ 0x53504152u /* "SPAR" */, (uint32_t)(seed >> 32));
    const int dl = synth_doc_len(g, key);
    uint32_t* tok = s_tok[warp];
    for (int i0 = lane * 4; i0 < SY_MAX_LEN; i0 += 128) {
        uint4 rnd = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), (uint32_t)(i0 >> 2), 2u), key);
        tok[i0 + 0] = i0 + 0 < dl ? synth_term(u01(rnd.x), vmax_pow, inv_exp, vocab) : 0xFFFFFFFFu;
        tok[i0 + 1] = i0 + 1 < dl ? synth_term(u01(rnd.y), vmax_pow, inv_exp, vocab) : 0xFFFFFFFFu;
        tok[i0 + 2] = i0 + 2 < dl ? synth_term(u01(rnd.z), vmax_pow, inv_exp, vocab) : 0xFFFFFFFFu;
        tok[i0 + 3] = i0 + 3 < dl ? synth_term(u01(rnd.w), vmax_pow, inv_exp, vocab) : 0xFFFFFFFFu;
    }
    __syncwarp();
    // warp bitonic sort of 512 tokens
    for (int k = 2; k <= SY_MAX_LEN; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = lane; t < SY_MAX_LEN / 2; t += 32) {
                int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                int p = i | j;
                bool up = ((i & k) == 0);
                uint32_t a = tok[i], b = tok[p];
                if ((a > b) == up) { tok[i] = b; tok[p] = a; }
            }
            __syncwarp();
        }
    }
    // run-length encode: a run starts at i when tok[i] != tok[i-1]
    int64_t base = MODE == 1 ? offsets[d] : 0;
    int runs_before = 0;
    for (int i0 = 0; i0 < SY_MAX_LEN; i0 += 32) {
        int i = i0 + lane;
        bool valid = i < dl;
        bool start = valid && (i == 0 || tok[i] != tok[i - 1]);
        unsigned m = __ballot_sync(0xffffffffu, start);
        if (MODE == 1 && start) {
            int pos = runs_before + __popc(m & ((1u << lane) - 1u));
            int e = i + 1;
            while (e < dl && tok[e] == tok[i]) ++e;
            term_ids[base + pos] = tok[i];
            term_tf[base + pos] = (uint16_t)(e - i);
        }
        runs_before += __popc(m);
    }
    if (MODE == 0 && lane == 0) { uniq[d] = runs_before; doc_len[d] = (uint32_t)dl; }
}

void synth_sparse(int64_t n, int64_t row_base, uint64_t seed, int64_t vocab, DevArray<int64_t>& offsets,
                  DevArray<uint32_t>& term_ids, DevArray<uint16_t>& term_tf, DevArray<uint32_t>& doc_len, int64_t* nnz_out,
                  cudaStream_t st)
{
    const float s = 1.07f;
    const float vmax_pow = powf((float)(vocab + 1), 1.f - s);
    const float inv_exp = 1.f / (1.f - s);
    DevArray<int64_t> uniq;
    uniq.alloc(n + 1);
    KRAG_CUDA(cudaMemsetAsync(uniq.p, 0, sizeof(int64_t) * (size_t)(n + 1), st));
    offsets.alloc(n + 1);
    doc_len.alloc(n > 0 ? n : 1);
    const unsigned grid = (unsigned)((n + SY_WARPS - 1) / SY_WARPS);
    if (n > 0) {
        synth_sparse_kernel<0><<<grid, SY_WARPS * 32, 0, st>>>(n, row_base, seed, vocab, vmax_pow, inv_exp, uniq.p, doc_len.p,
                                                               nullptr, nullptr, nullptr);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
    }
    size_t tmp_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, uniq.p, offsets.p, (int64_t)(n + 1), st);
    DevArray<unsigned char> tmp;
    tmp.alloc(tmp_bytes ? tmp_bytes : 16);
    cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, uniq.p, offsets.p, (int64_t)(n + 1), st);
    count_launch();
    int64_t nnz = 0;
    KRAG_CUDA(cudaMemcpyAsync(&nnz, offsets.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    KRAG_CUDA(cudaStreamSynchronize(st));
    tmp.release();
    uniq.release();
    term_ids.alloc(nnz > 0 ? nnz : 1);
    term_tf.alloc(nnz > 0 ? nnz : 1);
    if (n > 0) {
        synth_sparse_kernel<1><<<grid, SY_WARPS * 32, 0, st>>>(n, row_base, seed, vocab, vmax_pow, inv_exp, nullptr,
                                                               nullptr, offsets.p, term_ids.p, term_tf.p);
        KRAG_CUDA(cudaGetLastError());
        count_launch();
    }
    KRAG_CUDA(cudaStreamSynchronize(st));
    *nnz_out = nnz;
}

}  // namespace krag
