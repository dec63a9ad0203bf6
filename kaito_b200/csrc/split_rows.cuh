// split_rows.cuh -- the layout of device-resident fp32 rows with dpad % 64 == 0 ("split rows"); split_rows.cu holds its
// conversion kernels.  No other code knows the layout beyond the helpers below.
//
// A row of dpad fp32 values is dpad / 64 blocks of 256 bytes.  Block b holds elements [64 b, 64 b + 64): first their 64 high
// halves (128 B), then their 64 low halves (128 B).  For a value with bits x (u32):
//   hi = (x >> 16) + ((x & 0xFFFF) > 0x8000)     bf16 of x rounded to nearest, ties toward zero
//   lo = x & 0xFFFF
//   x  = ((hi - (lo > 0x8000)) << 16) | lo
// Ties go toward zero (not to even) so that the decode is unambiguous at lo == 0x8000.  hi is a bf16 within half a bf16 ulp of
// x, so the prune pass of K2 streams only the high halves (2 bytes per element, no extra memory) with the error bound of
// bf16 operands; every exact consumer (K1, rescoring, read-back, snapshots) rebuilds x bit for bit.  Every 32-bit pattern
// round-trips (the arithmetic is modulo 2^32).  A row keeps 4 * dpad bytes, so row moves (compaction, redeal) copy it
// unchanged.  Host-resident rows and indexes with dpad % 64 == 32 keep plain fp32 rows.
//
// Inside each half of a block the elements are in lane order: position 8 l + 4 h + c holds element 32 h + 4 l + c
// (l = 0..7, h = 0..1, c = 0..3).  These are the elements K1's lane l owns at its steps 2 b and 2 b + 1 (it sums elements
// 32 i + 4 l + c at step i), so each lane reads them as one 16-byte word of high halves and one of low halves.  A dot product
// over a block is the same in either order: K2's bf16 pass takes its queries in the same order (launch_bf16_split_order), and
// its TF32 pass gathers its fragments in element order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "common.cuh"

namespace krag {

constexpr int SPLIT_BLOCK = 64;   // elements per block: 128 B of high halves, then 128 B of low halves

__host__ __device__ __forceinline__ bool split_rows_layout(int dpad, bool host_rows) { return !host_rows && dpad % SPLIT_BLOCK == 0; }
__host__ __device__ __forceinline__ uint32_t split_hi(uint32_t x) { return ((x >> 16) + ((x & 0xFFFFu) > 0x8000u)) & 0xFFFFu; }
__host__ __device__ __forceinline__ uint32_t split_join(uint32_t hi, uint32_t lo) { return ((hi - (lo > 0x8000u)) << 16) | lo; }
// position inside a half-block of element e (0..63) of the block, and its inverse
__host__ __device__ __forceinline__ int split_pos(int e) { return 8 * ((e & 31) >> 2) + 4 * (e >> 5) + (e & 3); }
__host__ __device__ __forceinline__ int split_elem(int p) { return 32 * ((p >> 2) & 1) + 4 * (p >> 3) + (p & 3); }
// TMA view of split rows as 128-byte pieces of 64 halves: the high halves of block b are piece 2 b, the low halves 2 b + 1
__host__ __device__ __forceinline__ int split_pieces(int dpad) { return 2 * (dpad / SPLIT_BLOCK); }

__device__ __forceinline__ float4 split_decode4(uint2 hi, uint2 lo)
{
    return make_float4(__uint_as_float(split_join(hi.x & 0xFFFFu, lo.x & 0xFFFFu)), __uint_as_float(split_join(hi.x >> 16, lo.x >> 16)),
                       __uint_as_float(split_join(hi.y & 0xFFFFu, lo.y & 0xFFFFu)), __uint_as_float(split_join(hi.y >> 16, lo.y >> 16)));
}
// K1 lane l8's elements of block b of a split row: s0 = elements 64 b + 4 l8 + c (its step 2 b), s1 = 64 b + 32 + 4 l8 + c
// (step 2 b + 1).  STREAM: L1 no-allocate (the scan reads every row once); otherwise the read-only path.
template <bool STREAM>
__device__ __forceinline__ void split_ld8(const float* row, int b, int l8, float4& s0, float4& s1)
{
    const uint4* p = reinterpret_cast<const uint4*>(row + b * SPLIT_BLOCK) + l8;
    uint4 h, l;
    if (STREAM) {
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(h.x), "=r"(h.y), "=r"(h.z), "=r"(h.w) : "l"(p));
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(l.x), "=r"(l.y), "=r"(l.z), "=r"(l.w) : "l"(p + 8));
    } else {
        h = __ldg(p);
        l = __ldg(p + 8);
    }
    s0 = split_decode4(make_uint2(h.x, h.y), make_uint2(l.x, l.y));
    s1 = split_decode4(make_uint2(h.z, h.w), make_uint2(l.z, l.w));
}

// rows [0, n) of dpad elements at X, in place: plain fp32 -> split rows
void launch_split_encode(float* X, int64_t n, int dpad, cudaStream_t st);
// split rows [0, n) -> their values rounded to nearest-even bf16, plain row-major [n, dpad] (the KRAG_DENSE_TC_BF16 shadow)
void launch_split_to_bf16(const float* X, int64_t n, int dpad, uint16_t* out, cudaStream_t st);
// plain fp32 rows [n_elems / dpad, dpad] -> nearest-even bf16 with each 64-element block in the split rows' lane order
// (the query operand of K2's bf16 pass over split rows)
void launch_bf16_split_order(const float* in, uint16_t* out, int64_t n_elems, cudaStream_t st);

// the first `dim` fp32 values of one split row, on the host
inline void split_row_decode_host(const float* row, int dim, float* out)
{
    const uint16_t* h = reinterpret_cast<const uint16_t*>(row);
    for (int e = 0; e < dim; ++e) {
        const uint16_t* blk = h + (e / SPLIT_BLOCK) * 2 * SPLIT_BLOCK;
        const int p = split_pos(e % SPLIT_BLOCK);
        const uint32_t x = split_join(blk[p], blk[SPLIT_BLOCK + p]);
        memcpy(out + e, &x, 4);
    }
}

}  // namespace krag
