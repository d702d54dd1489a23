// K4: IGLOO patch gather, K6: attention softmax + weighted sum of the pooled projections.
//
// Reference semantics (genomad/neural_network/igloo.py:190-217):
//   M   = gather_nd(transpose(y), patches)                 -> y[b, P[p,k], c]
//   mpi = sum_k sum_c y[b,P[p,k],c] * w_mult[p,k,c] * w_summer[128k+c] + w_bias[p]      (lines 192-206)
//   alpha = softmax(mpi @ w_qk)   (lines 211-212; the GEMM is K5 in dense.cuh)
//   out = alpha @ maxpool8(y @ w_v)                        (lines 213-214)
// The patch weights are folded once at load time: Wf[p,k,c] = w_mult[p,k,c] * w_summer[128k+c]
// (fp32 product, so where the reference's two-step product underflows to 0, so does this one).
#pragma once
#include "common.cuh"

namespace gnm {

// ------------------------------------------------------------------------------------------
// Patch gather, position-ordered streaming form.
//
// The 8400 (patch, slot) entries of an IGLOO kernel touch only ~4500 distinct positions, so reading one
// row per entry moves every popular row ~1.9x through L2 -> SM.  Here the entries are sorted by position on the host and dealt to
// 700 CTAs x 4 warps x 3 entries (= 8400 exactly; 5 CTAs per SM, one resident wave, no shared memory): a warp's
// rows are neighbours in memory, repeats of a row are served by L1, and the whole grid sweeps each window
// front to back.  Every lane keeps its 3 x 8 folded weights in registers and a 3-window deep ring of
// row fragments in flight (one 512-byte row = ONE 16-byte load per lane: lanes 0-15 the fp16 "hi"
// half-row, lanes 16-31 the "lo" half-row; lanes l and l+16 use the same weights, so hi*w and lo*w meet
// in the warp-shuffle reduction).  Ahead of the ring, lanes 0-11 issue one prefetch.global.L2 each per window (the
// twelve 128-byte lines of the warp's three rows, kGsPrefetch windows further on): DRAM fetches start early at no
// register cost and the ring's loads mostly hit L2.  Each entry has exactly one writer (part[w][slot]);
// patch_finish_kernel then adds the four slots of a patch in fixed order k = 0..3 plus the bias, so results are
// deterministic.
// HBM-bound: 2.4 MB of distinct activation rows per window per IGLOO kernel (algorithmic 8400 x 512 B = 4.3 MB).
// ------------------------------------------------------------------------------------------
constexpr int kGsPerWarp = 3;                                    // entries per warp
constexpr int kGsThreads = 128;
constexpr int kGsPerCta = 4 * kGsPerWarp;                        // 12
constexpr int kGsGroups = (kPatches * kPatchLen + kGsPerCta - 1) / kGsPerCta;   // 700 CTAs (5 per SM, one wave)
constexpr int kGsSlots = kGsGroups * kGsPerCta;                  // 8400 (any remainder would be zero-weight padding)
constexpr int kGsDepth = 3;                                      // windows in flight per warp (registers)
constexpr int kGsPrefetch = 4;                                   // further windows requested into L2 ahead of the ring
constexpr int kGsMinBlocks = 5;
static_assert(kGsSlots >= kPatches * kPatchLen, "not enough entry slots");

__global__ void __launch_bounds__(kGsThreads, kGsMinBlocks)
patch_stream_kernel(const uint8_t* __restrict__ y,         // [n][5997][768 B]; reads the hi16 / lo16 planes (scaled by 32)
                    const int32_t* __restrict__ ent_pos,   // [kGsSlots] position of each slot (0 for padding)
                    const float* __restrict__ ent_w,       // [kGsSlots][128] folded weights / 32 of each slot (0 for padding)
                    float* __restrict__ part,              // [n][kGsSlots]
                    int n_windows) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = lane >> 4, l16 = lane & 15;
  const int e0 = blockIdx.x * kGsPerCta + warp * kGsPerWarp;
  int rowoff[kGsPerWarp];
  float wt[kGsPerWarp][8];
#pragma unroll
  for (int i = 0; i < kGsPerWarp; ++i) {
    rowoff[i] = ent_pos[e0 + i] * kRowBytes + (half ? kOffLo16 : kOffHi16) + l16 * 16;
    const float4 a = *reinterpret_cast<const float4*>(ent_w + static_cast<size_t>(e0 + i) * kC + l16 * 8);
    const float4 b = *reinterpret_cast<const float4*>(ent_w + static_cast<size_t>(e0 + i) * kC + l16 * 8 + 4);
    wt[i][0] = a.x; wt[i][1] = a.y; wt[i][2] = a.z; wt[i][3] = a.w;
    wt[i][4] = b.x; wt[i][5] = b.y; wt[i][6] = b.z; wt[i][7] = b.w;
  }
  const uint8_t* ybase = y;
  constexpr size_t kWinBytes = static_cast<size_t>(kTok) * kRowBytes;
  // L2 prefetch kGsPrefetch windows ahead of the register ring: the first 4 * kGsPerWarp lanes each own one 128-byte
  // line of the warp's 512-byte rows.
  const int pf_off = lane < 4 * kGsPerWarp ? ent_pos[e0 + (lane >> 2)] * kRowBytes + kOffHi16 + (lane & 3) * 128 : -1;
  if (pf_off >= 0)
    for (int d = kGsDepth; d < kGsDepth + kGsPrefetch && d < n_windows; ++d)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(ybase + d * kWinBytes + pf_off));
  uint4 ring[kGsDepth][kGsPerWarp];
#pragma unroll
  for (int d = 0; d < kGsDepth; ++d)
    if (d < n_windows) {
#pragma unroll
      for (int i = 0; i < kGsPerWarp; ++i)
        ring[d][i] = __ldg(reinterpret_cast<const uint4*>(ybase + d * kWinBytes + rowoff[i]));
    }
  for (int w0 = 0; w0 < n_windows; w0 += kGsDepth) {
#pragma unroll
    for (int d = 0; d < kGsDepth; ++d) {
      const int w = w0 + d;
      if (w < n_windows) {
        float acc[kGsPerWarp];
#pragma unroll
        for (int i = 0; i < kGsPerWarp; ++i) {
          const __half2* h = reinterpret_cast<const __half2*>(&ring[d][i]);
          float a = __low2float(h[0]) * wt[i][0];
          a = fmaf(__high2float(h[0]), wt[i][1], a);
          a = fmaf(__low2float(h[1]), wt[i][2], a); a = fmaf(__high2float(h[1]), wt[i][3], a);
          a = fmaf(__low2float(h[2]), wt[i][4], a); a = fmaf(__high2float(h[2]), wt[i][5], a);
          a = fmaf(__low2float(h[3]), wt[i][6], a); a = fmaf(__high2float(h[3]), wt[i][7], a);
          acc[i] = a;
        }
        if (w + kGsDepth < n_windows) {
#pragma unroll
          for (int i = 0; i < kGsPerWarp; ++i)
            ring[d][i] = __ldg(reinterpret_cast<const uint4*>(ybase + (w + kGsDepth) * kWinBytes + rowoff[i]));
        }
        if (pf_off >= 0 && w + kGsDepth + kGsPrefetch < n_windows)
          asm volatile("prefetch.global.L2 [%0];" ::"l"(ybase + (w + kGsDepth + kGsPrefetch) * kWinBytes + pf_off));
#pragma unroll
        for (int off = 16; off > 0; off >>= 1)
#pragma unroll
          for (int i = 0; i < kGsPerWarp; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
        if (lane < kGsPerWarp) {
          float r = acc[0];
#pragma unroll
          for (int i = 1; i < kGsPerWarp; ++i) r = lane == i ? acc[i] : r;
          part[static_cast<size_t>(w) * kGsSlots + e0 + lane] = r;
        }
      }
    }
  }
}

// mpi[w][p] = ((part[s0] + part[s1]) + part[s2]) + part[s3] + bias[p],  s_k = slot_of[4p + k]
// Also writes the value's two TF32 halves (hi + lo, low 13 mantissa bits clear) for the tensor-core logits GEMM (logits_tc.cuh).
__global__ void __launch_bounds__(256)
patch_finish_kernel(const float* __restrict__ part, const int32_t* __restrict__ slot_of, const float* __restrict__ w_bias,
                    float* __restrict__ mpi, float* __restrict__ mpi_hi, float* __restrict__ mpi_lo, int n_windows) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int w = blockIdx.y;
  if (p >= kPatches) return;
  const float* pw = part + static_cast<size_t>(w) * kGsSlots;
  const int4 s4 = *reinterpret_cast<const int4*>(slot_of + p * 4);
  const float v = (((pw[s4.x] + pw[s4.y]) + pw[s4.z]) + pw[s4.w]) + w_bias[p];
  const size_t o = static_cast<size_t>(w) * kPatches + p;
  mpi[o] = v;
  const float hi = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
  mpi_hi[o] = hi;
  mpi_lo[o] = __uint_as_float(__float_as_uint(v - hi) & 0xffffe000u);
}

// ------------------------------------------------------------------------------------------
// Attention tail: one CTA (128 threads = channels) per (window, igloo).  Row softmax over the
// 749 logits (max-subtracted, expf, fp32), then out[c] = sum_g alpha[g] * q[g][c].
// ------------------------------------------------------------------------------------------
constexpr int kLogitsLd = 752;     // logits row stride (749 rounded up to a multiple of 4)

__global__ void __launch_bounds__(128)
attention_kernel(const float* __restrict__ logits,   // [n][752]
                 const float* __restrict__ q,        // [n][749][128]
                 float* __restrict__ h0,             // [n][256]
                 float* __restrict__ h0_hi, float* __restrict__ h0_lo,   // TF32 halves of h0 for the tensor-core head (or nullptr)
                 int col_offset) {                   // 0 for IGLOO#0, 128 for IGLOO#1
  __shared__ float s_alpha[kPooled];
  __shared__ float s_red[4];
  const int w = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* lrow = logits + static_cast<size_t>(w) * kLogitsLd;
  float m = -INFINITY;
  for (int g = tid; g < kPooled; g += 128) { const float v = lrow[g]; s_alpha[g] = v; m = fmaxf(m, v); }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if (lane == 0) s_red[warp] = m;
  __syncthreads();
  m = fmaxf(fmaxf(s_red[0], s_red[1]), fmaxf(s_red[2], s_red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int g = tid; g < kPooled; g += 128) { const float e = expf(s_alpha[g] - m); s_alpha[g] = e; sum += e; }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  if (lane == 0) s_red[warp] = sum;
  __syncthreads();
  sum = (s_red[0] + s_red[1]) + (s_red[2] + s_red[3]);
  const float inv = 1.f / sum;
  const float* qw = q + static_cast<size_t>(w) * kPooled * kC + tid;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int g = 0;
  for (; g + 4 <= kPooled; g += 4) {
    a0 = fmaf(s_alpha[g] * inv, qw[static_cast<size_t>(g) * kC], a0);
    a1 = fmaf(s_alpha[g + 1] * inv, qw[static_cast<size_t>(g + 1) * kC], a1);
    a2 = fmaf(s_alpha[g + 2] * inv, qw[static_cast<size_t>(g + 2) * kC], a2);
    a3 = fmaf(s_alpha[g + 3] * inv, qw[static_cast<size_t>(g + 3) * kC], a3);
  }
  for (; g < kPooled; ++g) a0 = fmaf(s_alpha[g] * inv, qw[static_cast<size_t>(g) * kC], a0);
  const float v = (a0 + a1) + (a2 + a3);
  const size_t o = static_cast<size_t>(w) * 256 + col_offset + tid;
  h0[o] = v;
  if (h0_hi) {
    const float hi = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
    h0_hi[o] = hi;
    h0_lo[o] = __uint_as_float(__float_as_uint(v - hi) & 0xffffe000u);
  }
}

}  // namespace gnm
