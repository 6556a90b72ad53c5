// Warp-level tensor-core building blocks (mma.sync, ldmatrix, cp.async, shared-memory access by 32-bit address) and
// the split-bf16 rule, shared by the kernels of the library.  tc_common.cuh includes this header.
#pragma once
#include <cuda_bf16.h>

#include <cstdint>

namespace mm {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- split-bf16: the library's fp32-grade operand format, x = hi + lo with hi = bf16(x), lo = bf16(x - hi).
// Products run as hi*lo + lo*hi + hi*hi with fp32 accumulation.  Operand rows split ahead of time (mm_split_rows,
// the table mirrors, the tower epilogues) and rows split inside a kernel give bit-identical results only because
// every producer rounds exactly like this.
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
// (x, y) -> packed bf16x2 hi (x in the low half: K element 2c in the low 16 bits) and the bf16x2 of the residuals
__device__ __forceinline__ void split_pair(float x, float y, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  const float xh = __uint_as_float(hi << 16), yh = __uint_as_float(hi & 0xffff0000u);
  __nv_bfloat162 l = __floats2bfloat162_rn(x - xh, y - yh);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

// ---- c (16 x 8, fp32) += a (16 x 16 bf16, row-major fragment) . b (16 x 8 bf16, column-major fragment)
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---- ldmatrix: four 8 x 8 b16 matrices, lane l supplies the row address of row (l & 7) of matrix (l >> 3)
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}

// ---- cp.async, predicated in PTX: no branch / reconvergence bookkeeping around the copy
__device__ __forceinline__ void cp_async16_if(bool pred, uint32_t dst, const void* src) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p cp.async.cg.shared.global [%0], [%1], 16;\n\t}" ::"r"(dst),
      "l"(src), "r"((uint32_t)pred)
      : "memory");
}
__device__ __forceinline__ void cp_async4_if(bool pred, uint32_t dst, const void* src) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p cp.async.ca.shared.global [%0], [%1], 4;\n\t}" ::"r"(dst),
      "l"(src), "r"((uint32_t)pred)
      : "memory");
}
// 4- / 8-byte cp.async that writes zeros instead of copying when !valid (src-size 0: nothing is read from src)
__device__ __forceinline__ void cp_async4_zfill(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(valid ? 4u : 0u) : "memory");
}
__device__ __forceinline__ void cp_async8_zfill(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(valid ? 8u : 0u) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

}  // namespace mm
