// Warpgroup tensor-core MMA (wgmma, sm_90a): D[64 x N] (+)= A[64 x K] * B[K x N] with both operands in shared memory
// (K-major, 128-byte swizzle, see gmma_desc_sw128) and the fp32 accumulator in the registers of the issuing warpgroup.
// Accumulator fragment of thread t of the warpgroup (warp w = t / 32, lane l = t % 32), register i < N / 2:
//     row = 16 w + l / 4 + 8 ((i >> 1) & 1),   column = 8 (i >> 2) + 2 (l % 4) + (i & 1).
// The wrappers below are one instruction each; `accumulate` = 0 overwrites the accumulator.
#pragma once
#include <stdint.h>

namespace gnm {

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending> __device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// keeps the compiler from moving reads of the accumulator registers above wgmma_wait
template <int kN> __device__ __forceinline__ void wgmma_fence_regs(float (&d)[kN]) {
#pragma unroll
  for (int i = 0; i < kN; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor, K-major operand, SWIZZLE_128B, 8-row groups 1024 B apart.
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4 (unused for swizzled K-major; 1)
//   bits [32,46) stride byte offset >> 4   bits [49,52) base offset = 0 (slabs are 1024 B aligned)
//   bits [62,64) layout type (1 = SWIZZLE_128B)
// The swizzle is applied to the absolute shared-memory address, as TMA applies it when it fills a 1024 B aligned slab, so a
// descriptor may start at any 128-byte row of such a slab (the convolution taps and the K steps inside a row rely on it;
// the conv parity tests check it).
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

#define GNM_ACC8(b) "+f"(d[b]), "+f"(d[b + 1]), "+f"(d[b + 2]), "+f"(d[b + 3]), "+f"(d[b + 4]), "+f"(d[b + 5]), "+f"(d[b + 6]), "+f"(d[b + 7])
__device__ __forceinline__ void wgmma_f16_n48(float (&d)[24], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24,%25,p,1,1,0,0;\n}"
               : GNM_ACC8(0), GNM_ACC8(8), GNM_ACC8(16)
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16_n192(float (&d)[96], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %98, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}, %96,%97,p,1,1,0,0;\n}"
               : GNM_ACC8(0), GNM_ACC8(8), GNM_ACC8(16), GNM_ACC8(24), GNM_ACC8(32), GNM_ACC8(40), GNM_ACC8(48), GNM_ACC8(56), GNM_ACC8(64), GNM_ACC8(72), GNM_ACC8(80), GNM_ACC8(88)
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128,%129,p,1,1,0,0;\n}"
               : GNM_ACC8(0), GNM_ACC8(8), GNM_ACC8(16), GNM_ACC8(24), GNM_ACC8(32), GNM_ACC8(40), GNM_ACC8(48), GNM_ACC8(56), GNM_ACC8(64), GNM_ACC8(72), GNM_ACC8(80), GNM_ACC8(88), GNM_ACC8(96), GNM_ACC8(104), GNM_ACC8(112), GNM_ACC8(120)
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_e4m3_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n256k32.f32.e4m3.e4m3 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128,%129,p,1,1;\n}"
               : GNM_ACC8(0), GNM_ACC8(8), GNM_ACC8(16), GNM_ACC8(24), GNM_ACC8(32), GNM_ACC8(40), GNM_ACC8(48), GNM_ACC8(56), GNM_ACC8(64), GNM_ACC8(72), GNM_ACC8(80), GNM_ACC8(88), GNM_ACC8(96), GNM_ACC8(104), GNM_ACC8(112), GNM_ACC8(120)
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128,%129,p,1,1;\n}"
               : GNM_ACC8(0), GNM_ACC8(8), GNM_ACC8(16), GNM_ACC8(24), GNM_ACC8(32), GNM_ACC8(40), GNM_ACC8(48), GNM_ACC8(56), GNM_ACC8(64), GNM_ACC8(72), GNM_ACC8(80), GNM_ACC8(88), GNM_ACC8(96), GNM_ACC8(104), GNM_ACC8(112), GNM_ACC8(120)
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_n192(float (&d)[96], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %98, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n192k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}, %96,%97,p,1,1;\n}"
               : GNM_ACC8(0), GNM_ACC8(8), GNM_ACC8(16), GNM_ACC8(24), GNM_ACC8(32), GNM_ACC8(40), GNM_ACC8(48), GNM_ACC8(56), GNM_ACC8(64), GNM_ACC8(72), GNM_ACC8(80), GNM_ACC8(88)
               : "l"(da), "l"(db), "r"(accumulate));
}
#undef GNM_ACC8

}  // namespace gnm
