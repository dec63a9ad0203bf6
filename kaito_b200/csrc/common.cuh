// common.cuh -- shared device/host helpers for libkaito_rag (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#define KRAG_LANES 32  // fp32 partial sums per row; rows are zero-padded to a multiple of 32 floats

namespace krag {

// ---------------------------------------------------------------- error plumbing (host)
void set_error(const std::string& msg);
struct CudaError { cudaError_t e; const char* what; const char* file; int line; };
#define KRAG_CUDA(expr)                                                        \
    do {                                                                       \
        cudaError_t _e = (expr);                                               \
        if (_e != cudaSuccess) throw ::krag::CudaError{_e, #expr, __FILE__, __LINE__}; \
    } while (0)

// --------------------------------------------------------------------- candidate keys
// key = ordered_bits(value) << 32 | ordinal;  ascending key == (value asc, ordinal asc).
__host__ __device__ __forceinline__ uint32_t f32_ordered_bits(float f)
{
#ifdef __CUDA_ARCH__
    uint32_t u = __float_as_uint(f);
#else
    union { float f; uint32_t u; } c; c.f = f; uint32_t u = c.u;
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float f32_from_ordered_bits(uint32_t o)
{
    uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    union { float f; uint32_t u; } c; c.u = u; return c.f;
#endif
}
__host__ __device__ __forceinline__ uint64_t make_key_asc(float v, uint32_t ord)
{
    return ((uint64_t)f32_ordered_bits(v) << 32) | ord;
}
__host__ __device__ __forceinline__ uint64_t make_key_desc(float v, uint32_t ord)
{
    return ((uint64_t)(~f32_ordered_bits(v)) << 32) | ord;
}
__host__ __device__ __forceinline__ float key_value_asc(uint64_t k) { return f32_from_ordered_bits((uint32_t)(k >> 32)); }
__host__ __device__ __forceinline__ float key_value_desc(uint64_t k) { return f32_from_ordered_bits(~(uint32_t)(k >> 32)); }
__host__ __device__ __forceinline__ uint32_t key_ordinal(uint64_t k) { return (uint32_t)k; }

constexpr uint64_t KEY_PAD = 0xFFFFFFFFFFFFFFFFull;

__host__ __device__ __forceinline__ int next_pow2(int v)
{
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

#ifdef __CUDACC__
// ------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ float4 ldg_stream_f4(const float4* p)
{
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ldg_stream_u2(const uint2* p)
{
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
// named barrier over `nthreads` threads (id 0 with the full CTA == __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ bool bit_test(const uint32_t* __restrict__ bm, uint32_t i)
{
    return (bm[i >> 5] >> (i & 31)) & 1u;
}
#endif

}  // namespace krag
