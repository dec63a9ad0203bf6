// split_rows.cu -- conversion kernels of the split-row layout (split_rows.cuh).
#include <cuda_bf16.h>

#include "engine.h"
#include "split_rows.cuh"

namespace krag {

static unsigned conv_blocks(int64_t threads)
{
    const int64_t b = (threads + 255) / 256;
    return (unsigned)(b < 132 * 16 ? b : 132 * 16);
}

// in place, one warp per 64-element block (256 bytes): lane l takes positions 2 l and 2 l + 1, i.e. elements split_elem(2 l)
// and the next one; every lane reads before any lane of the warp writes
__global__ void __launch_bounds__(256) split_encode_kernel(uint32_t* __restrict__ X, int64_t n_blocks)
{
    const int lane = threadIdx.x & 31;
    const int64_t step = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n_blocks; b += step) {
        uint32_t* blk = X + b * SPLIT_BLOCK;
        const uint2 v = reinterpret_cast<const uint2*>(blk)[split_elem(2 * lane) / 2];
        const uint32_t hi = split_hi(v.x) | (split_hi(v.y) << 16), lo = (v.x & 0xFFFFu) | (v.y << 16);
        __syncwarp();
        blk[lane] = hi;
        blk[SPLIT_BLOCK / 2 + lane] = lo;
    }
}
void launch_split_encode(float* X, int64_t n, int dpad, cudaStream_t st)
{
    const int64_t n_blocks = n * (dpad / SPLIT_BLOCK);
    if (n_blocks == 0) return;
    split_encode_kernel<<<conv_blocks(n_blocks * 32), 256, 0, st>>>(reinterpret_cast<uint32_t*>(X), n_blocks);
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// one thread per word w of high halves (block w / 32, positions 2 l and 2 l + 1, l = w % 32)
__global__ void __launch_bounds__(256) split_to_bf16_kernel(const uint32_t* __restrict__ X, int64_t n_words, uint32_t* __restrict__ out)
{
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = w >> 5;
        const int l = (int)(w & 31);
        const uint32_t hi = X[b * SPLIT_BLOCK + l], lo = X[b * SPLIT_BLOCK + SPLIT_BLOCK / 2 + l];
        const __nv_bfloat162 v = __floats2bfloat162_rn(__uint_as_float(split_join(hi & 0xFFFFu, lo & 0xFFFFu)),
                                                       __uint_as_float(split_join(hi >> 16, lo >> 16)));
        out[(b * SPLIT_BLOCK + split_elem(2 * l)) / 2] = *reinterpret_cast<const uint32_t*>(&v);
    }
}
void launch_split_to_bf16(const float* X, int64_t n, int dpad, uint16_t* out, cudaStream_t st)
{
    const int64_t n_words = n * dpad / 2;
    if (n_words == 0) return;
    split_to_bf16_kernel<<<conv_blocks(n_words), 256, 0, st>>>(reinterpret_cast<const uint32_t*>(X), n_words,
                                                                reinterpret_cast<uint32_t*>(out));
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

// one thread per output pair (positions 2 l, 2 l + 1 of a block)
__global__ void __launch_bounds__(256) bf16_split_order_kernel(const float2* __restrict__ in, int64_t n_pairs, uint32_t* __restrict__ out)
{
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_pairs; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = w >> 5;
        const float2 v = in[(b * SPLIT_BLOCK + split_elem(2 * (int)(w & 31))) / 2];
        const __nv_bfloat162 h = __floats2bfloat162_rn(v.x, v.y);
        out[w] = *reinterpret_cast<const uint32_t*>(&h);
    }
}
void launch_bf16_split_order(const float* in, uint16_t* out, int64_t n_elems, cudaStream_t st)
{
    if (n_elems == 0) return;
    bf16_split_order_kernel<<<conv_blocks(n_elems / 2), 256, 0, st>>>(reinterpret_cast<const float2*>(in), n_elems / 2,
                                                                     reinterpret_cast<uint32_t*>(out));
    KRAG_CUDA(cudaGetLastError());
    count_launch();
}

}  // namespace krag
