// Shared device helpers for the geNomad kernels (sm_90a).
// Raw PTX wrappers for mbarrier / TMA (wgmma: wgmma.cuh) -- no CUTLASS, no Triton.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#include "wgmma.cuh"

namespace gnm {

// ----------------------------------------------------------------------------- model constants
constexpr int kWindow   = 6000;   // nucleotides per window            (reference nn_classification.py:68)
constexpr int kTok      = 5997;   // 4-mer tokens per window           (reference sequence.py:172)
constexpr int kVocab    = 257;    // one-hot depth                     (reference model.py:11)
constexpr int kC        = 128;    // conv filters                      (reference model.py:20)
constexpr int kTaps     = 6;      // conv kernel size                  (reference model.py:22)
constexpr int kPatches  = 2100;   // IGLOO patches                     (reference model.py:19)
constexpr int kPatchLen = 4;      // IGLOO patch size                  (reference igloo.py:34)
constexpr int kPool     = 8;      // max-pool size                     (reference model.py:23)
constexpr int kPooled   = 749;    // 5997 // 8                         (reference igloo.py:164)
constexpr int kHidden   = 512;    // dense width                       (reference model.py:28,40)
constexpr float kLeaky  = 0.1f;   // LeakyReLU slope                   (reference igloo.py:48,67)

// Activation row in HBM: 768 bytes per position.  With Y = 32 * y (kActScale keeps the fp16 "lo" part and the fp8
// planes away from their subnormal ranges).  Range: the e4m3 plane hi8 = hi16 * 4 saturates (SATFINITE, 448) once
// |Y| > 112, i.e. |y| > 3.5 -- the Ahi*Wlo correction pass of the next conv would then be wrong and precision would fall
// back to the single-pass level (~1.3e-4) -- and fp16 itself overflows at |y| > 2047.  Producers check both limits and raise
// DeviceStatus::act_overflow (reported by the next API call as an error); the shipped model stays below |y| = 0.7.
//   [  0,256)  hi16 = fp16(Y)                       128 halves   -- main tensor-core operand, w_v, patch gather
//   [256,512)  lo16 = fp16(Y - hi16)                128 halves   -- w_v 3-pass split, patch gather
//   [512,768)  p8   = 128 e4m3 PAIRS (lo8[c], hi8[c]),  lo8 = e4m3((Y - hi16) * 128), hi8 = e4m3(hi16 * 4)
//                     -- the operand of the convs' correction passes lo(A) * hi(W) + hi(A) * lo(W), which run as ONE K = 256
//                     contraction against weights interleaved the same way (Whi8[c], Wlo8[c]).  Interleaving (round 2) makes a
//                     channel's two bytes one b16 element (conv2's epilogue transposes this plane with the same b16 stmatrix
//                     as hi16; layer 1: one 8-byte store per lane instead of two 4-byte stores).
constexpr int kRowBytes  = 768;
constexpr int kOffHi16   = 0, kOffLo16 = 256, kOffP8 = 512;
constexpr float kActScale = 32.f;          // 2^5
constexpr float kLo8Scale = 128.f;         // lo8 = (Y - hi16) * 2^7   -> y_lo * 2^12
constexpr float kHi8Scale = 4.f;           // hi8 = hi16 * 2^2         -> y_hi * 2^7
constexpr float kHi8Limit = 448.f / kHi8Scale;   // |Y| above this saturates the hi8 plane   (|y| > 3.5)
constexpr float kF16Limit = 65504.f;             // |Y| above this overflows the hi16 plane  (|y| > 2047)

// ----------------------------------------------------------------------------- small utils
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ float lrelu(float x) { return x > 0.f ? x : x * kLeaky; }

// fp32 -> (hi, lo) fp16 pair with hi + lo ~= x to ~22 bits
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  hi = __float2half_rn(x);
  lo = __float2half_rn(x - __half2float(hi));
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  return static_cast<uint32_t>(__half_as_ushort(a)) | (static_cast<uint32_t>(__half_as_ushort(b)) << 16);
}

// Packed fp32 -> (hi, lo) fp16 split of two values: one F2FP pack for hi, one unpack, one F2FP pack for lo
// (the scalar F2F conversions run on the slow conversion pipe: 16/clk/SM).
__device__ __forceinline__ void split2_f16(float a, float b, __half2& hi, __half2& lo) {
  hi = __floats2half2_rn(a, b);
  const float2 f = __half22float2(hi);
  lo = __floats2half2_rn(a - f.x, b - f.y);
}

// two floats -> two e4m3 bytes (round to nearest even, saturating)
__device__ __forceinline__ uint16_t pack_e4m3x2(float a, float b) {
  return static_cast<uint16_t>(__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3));
}

// ----------------------------------------------------------------------------- shared-memory transposes
// Four 8x8 b16 matrices from an mma-style fragment (register i: matrix i; lane l holds row l / 4, columns 2 (l % 4) and
// 2 (l % 4) + 1, the lower column in the low half), stored TRANSPOSED: row r of matrix i (16 bytes) goes to the address lane
// 8 i + r passes, and holds column r of the fragment.
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t saddr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};"
               ::"r"(saddr), "r"(r0), "r"(r1), "r"(r2), "r"(r3) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr) : "memory");
  return v;
}

// error flag written by device-side timeouts (see mbar_wait); checked by the host API
struct DeviceStatus { int code; int info0; int info1; int info2; int act_overflow; int ov_stage[4]; };
enum : int { kDevOk = 0, kDevMbarTimeout = 1 };
// activation range check (see the row layout above): stage = 1 layer 1, 2 conv2, 3 conv3
__device__ __forceinline__ void flag_act_overflow(DeviceStatus* st, float absmax, float limit, int stage) {
  if (absmax > limit && st) { st->act_overflow = 1; st->ov_stage[stage] = 1; }
}

// exactly one lane of a fully converged warp gets true (PTX elect.sync); ptxas then keeps the
// guarded TMA instructions on the uniform datapath instead of a per-lane waterfall loop
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  // The fourth operand is the suspend-time hint (ns): the waiting thread is parked in hardware until the phase completes or
  // the hint expires.  Without it a waiter wakes every few hundred cycles and re-issues the whole spin loop -- ncu on the
  // fused IGLOO kernel counted ~60 try_waits per warp and unit, i.e. a fifth of all issued instructions in a kernel
  // whose consumer warps are short of issue slots.
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(20000u) : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must become a CUDA error, never a hung GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, DeviceStatus* st, int tag) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  for (uint32_t spins = 1;; ++spins) {
    if (mbar_try_wait(bar, parity)) return;          // try_wait itself suspends the thread for a hardware-defined time slice
    if ((spins & 255u) == 0 && clock64() - t0 > 4000000000LL) {   // ~2 s at 2 GHz; the clock is read once per 256 spins
      if (st) { st->code = kDevMbarTimeout; st->info0 = tag; st->info1 = blockIdx.x; st->info2 = threadIdx.x; }
      __threadfence_system();
      __trap();
    }
  }
}

// ----------------------------------------------------------------------------- TMA (cp.async.bulk.tensor)
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// L2 eviction-priority policies for TMA loads (weights are re-read by every CTA: keep; activations stream through once)
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_hint(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(policy)
      : "memory");
}
}  // namespace gnm
