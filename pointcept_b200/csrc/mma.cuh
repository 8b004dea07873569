// Thin inline-PTX layer over the Hopper (sm_90a) warp-level tensor-core path: mma.sync m16n8k16 (fp16 / bf16 in, fp32
// accumulate), ldmatrix and cp.async.
//
// Fragment layouts of mma.m16n8k16 (g = lane / 4, t = lane % 4), the contract every kernel of this library relies on:
//   A (16 x 16, row-major)  a[0] = (row g,   k 2t..2t+1)   a[1] = (row g+8, k 2t..2t+1)
//                           a[2] = (row g,   k 2t+8..+9)   a[3] = (row g+8, k 2t+8..+9)
//   B (16 x 8)              b[0] = (k 2t..2t+1, col g)     b[1] = (k 2t+8..+9, col g)
//   C / D (16 x 8, fp32)    d[0..1] = (row g, col 2t..2t+1)  d[2..3] = (row g+8, col 2t..2t+1)
// so the accumulator of two adjacent 8-column tiles, rounded to 16 bit, is the A fragment of a 16-deep K step (P V in attention).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace b2pc {
namespace mma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- cp.async (16- / 4-byte pieces, zero fill when !valid) -----------------------------------------------------------------
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t smem_dst, const void* gsrc, bool valid) {
  const int sz = valid ? 4 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- ldmatrix: four 8 x 8 matrices of 16-bit elements; lane l supplies the address of row l % 8 of matrix l / 8 ------------
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

// ---- D (+)= A B on the tensor cores ------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (std::is_same<T, __nv_bfloat16>::value) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

// ---- shared-memory tile addressing --------------------------------------------------------------------------------------------
// Rows of 16 channels (32 bytes, head_dim 16): the two 16-byte halves of row r swap places when bit 2 of r is set, so the eight rows
// an ldmatrix phase reads fall on eight distinct 16-byte bank groups.
__device__ __forceinline__ uint32_t row32_off(int r, int half) { return (uint32_t)(r * 32 + (((half ^ (r >> 2)) & 1) << 4)); }

// lane -> (row, column) of the 16 x 16 block an ldmatrix.x4 reads, for the three fragment kinds used here
//   A from row-major [m][k] (non-trans):    m = l % 16,             k = (l / 16) * 8
//   B from [n][k] (non-trans, two 8-col tiles): n = l % 8 + (l / 16) * 8,  k = ((l / 8) % 2) * 8
//   B from [k][n] (trans, two 8-col tiles):     k = l % 8 + ((l / 8) % 2) * 8,  n = (l / 16) * 8
//   A from [k][m] (trans):                  k = l % 8 + (l / 16) * 8,  m = ((l / 8) % 2) * 8
struct LdsmA   { __device__ static int r(int l) { return l & 15; }                       __device__ static int c(int l) { return (l >> 4) << 3; } };
struct LdsmBnk { __device__ static int r(int l) { return (l & 7) + ((l >> 4) << 3); }    __device__ static int c(int l) { return ((l >> 3) & 1) << 3; } };
struct LdsmBkn { __device__ static int r(int l) { return (l & 7) + (((l >> 3) & 1) << 3); } __device__ static int c(int l) { return (l >> 4) << 3; } };
struct LdsmAkm { __device__ static int r(int l) { return (l & 7) + ((l >> 4) << 3); }    __device__ static int c(int l) { return ((l >> 3) & 1) << 3; } };

// ---- misc ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

}  // namespace mma

template <typename T> __device__ __forceinline__ uint32_t pack2(float lo, float hi);
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

}  // namespace b2pc
