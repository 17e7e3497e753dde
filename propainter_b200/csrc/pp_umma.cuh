// wgmma / mbarrier building blocks (sm_90a); operands K-major SWIZZLE_128B (TF32 wgmma needs K-major).  Accumulator of
// m64nN: warp w holds rows 16w + g, 16w + g + 8 (g = lane / 4), columns 8j + 2(lane % 4) + {0, 1} in d[4j + {0,1} / {2,3}].
// All mbarrier waits are bounded and trap instead of hanging.
#pragma once
#include <cstdint>

__device__ __forceinline__ uint32_t ua_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ua_bar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void ua_bar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void ua_bar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (int spin = 0; spin < (1 << 26) && !done; ++spin)
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  if (!done) __trap();
}
// one lane of the (converged) warp: lets ptxas keep TMA operands in uniform registers and predicate the single
// instruction, instead of looping over the active lanes of a divergent region
__device__ __forceinline__ bool ua_elect() {
  uint32_t pred = 0;
  asm volatile("{ .reg .b32 r; .reg .pred p; elect.sync r|p, 0xffffffff; selp.u32 %0, 1, 0, p; }" : "=r"(pred));
  return pred != 0;
}
// K-major SWIZZLE_128B shared-memory matrix descriptor (LBO unused = 16 B, SBO = 1024 B between 8-row groups, layout 1 = 128B swizzle)
__device__ __forceinline__ uint64_t ua_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// byte offset of element (row, k) in a K-major SW128 tile with `rows` rows: k-block (32 floats) major, 8-row groups of 1 KB
__device__ __forceinline__ uint32_t ua_off(int row, int k, int rows) {
  const int kb = k >> 5, kk = k & 31, r = row & 7;
  return (uint32_t)(kb * rows * 128 + (row >> 3) * 1024 + r * 128 + (((kk >> 2) ^ r) << 4) + (kk & 3) * 4);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// wgmma writes its accumulator registers asynchronously: pin them around wg_wait with wg_pin (an empty volatile asm per
// register), so the compiler does not move their reads or writes across the wait; issue wg_fence() before the next wgmma.
template <int R>
__device__ __forceinline__ void wg_pin(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
#define WG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wg_mma_ss_n32(float (&d)[16], uint64_t a, uint64_t b, int scale_d) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %18, 0; wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1; }"
               : WG_D8(0), WG_D8(8)
               : "l"(a), "l"(b), "r"(scale_d));
}

__device__ __forceinline__ void wg_mma_ss_n64(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %34, 0; wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1; }"
               : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24)
               : "l"(a), "l"(b), "r"(scale_d));
}

__device__ __forceinline__ void wg_mma_ss_n128(float (&d)[64], uint64_t a, uint64_t b, int scale_d) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %66, 0; wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1; }"
               : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24), WG_D8(32), WG_D8(40), WG_D8(48), WG_D8(56)
               : "l"(a), "l"(b), "r"(scale_d));
}

__device__ __forceinline__ void wg_mma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t b, int scale_d) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %69, 0; wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1; }"
               : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24), WG_D8(32), WG_D8(40), WG_D8(48), WG_D8(56)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}

// ---- 16-bit operands (f32 += f16 x f16, k16 per instruction).  A K-major SW128 tile holds 64 halves per 128-byte row, so a
// k16 step is the same 32-byte advance as a tf32 k8 step.  An MN-major B (imm-trans-b = 1) is read from rows = K, 64 N-elements
// per 128-byte row, 8-row swizzle atoms SBO = 1024 B apart along K and 64-element N blocks LBO = `lbo` bytes apart.
__device__ __forceinline__ uint64_t ua_desc_mn(uint32_t saddr, uint32_t lbo) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wg_mma_ss_n32_f16(float (&d)[16], uint64_t a, uint64_t b, int scale_d) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %18, 0; wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0; }"
               : WG_D8(0), WG_D8(8)
               : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wg_mma_ss_n64_f16(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %34, 0; wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0; }"
               : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24)
               : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wg_mma_ss_n128_f16(float (&d)[64], uint64_t a, uint64_t b, int scale_d) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %66, 0; wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0; }"
               : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24), WG_D8(32), WG_D8(40), WG_D8(48), WG_D8(56)
               : "l"(a), "l"(b), "r"(scale_d));
}
// A from registers (4 x half2 per thread: rows g / g + 8, k 2t..2t+1 / 2t+8..2t+9), B MN-major
__device__ __forceinline__ void wg_mma_rs_n128_f16_tb(float (&d)[64], const uint32_t (&a)[4], uint64_t b, int scale_d) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %69, 0; wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 1; }"
               : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24), WG_D8(32), WG_D8(40), WG_D8(48), WG_D8(56)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
