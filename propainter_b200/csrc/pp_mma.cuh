// Warp-level TF32 tensor-core helpers (mma.sync m16n8k8, fp32 accumulate) + cp.async.
//
// Fragment ownership for lane = 4*g + t (g = 0..7, t = 0..3):
//   A (16x8 row-major)  a0=(g,t) a1=(g+8,t) a2=(g,t+4) a3=(g+8,t+4)
//   B (8x8  col-major)  b0=(k=t,n=g) b1=(k=t+4,n=g)
//   C (16x8)            c0=(g,2t) c1=(g,2t+1) c2=(g+8,2t) c3=(g+8,2t+1)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

__device__ __forceinline__ uint32_t pp_tf32(float f) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(f));
  return r;
}
__device__ __forceinline__ void pp_mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// D += A(16x16, f16, row) * B(16x8, f16, col), fp32 accumulate: a = rows g / g+8 x k 2t..2t+1 / 2t+8..2t+9, b = k 2t..2t+1 /
// 2t+8..2t+9 x n g, packed half2
__device__ __forceinline__ void pp_mma_f16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// four transposed 8x8 b16 matrices; lane l supplies the address of row l % 8 of matrix l / 8
__device__ __forceinline__ void pp_ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void pp_cp_async16(void* smem, const void* gmem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void pp_cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void pp_cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }
