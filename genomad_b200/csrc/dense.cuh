// K5 (attention logits GEMM), K7 (dense head) and K8 (per-contig segment reduction).
//
// Reference semantics:
//   alpha logits = mpi @ w_qk                      genomad/neural_network/igloo.py:211
//   Dense(512)+BatchNormalization+relu             genomad/neural_network/model.py:28-30, 40-42
//         keras BN inference: x * inv + (beta - mean * inv), inv = gamma * rsqrt(var + 1e-3)
//   Dense(3, softmax)                              genomad/neural_network/model.py:44
//   tf.math.segment_mean(preds, contig_ids)        genomad/modules/nn_classification.py:320
#pragma once
#include "common.cuh"

namespace gnm {

// ------------------------------------------------------------------------------------------
// C[M][ldc] = epi(A[M][K] @ B[K][N]) in fp32 on the CUDA cores (these GEMMs are < 0.3 % of the
// model's FLOPs).  16-deep K slices, (4x4) outputs per thread, guards on every edge.  Each output element
// is accumulated in k order by one thread, so results do not depend on the tile shape or batch position.
// epi: v = acc + bias[n]; if scale: v = v * scale[n] + shift[n]; if relu: v = max(v, 0).
// ------------------------------------------------------------------------------------------
constexpr int kGemmBN = 64, kGemmBK = 16;

// kBM x 64 output tile per CTA (kBM = 32 or 64; kBM*4 threads, 4x4 outputs each).  The 32-row variant is used when
// the 64-row grid would leave SMs idle (M = 1024 windows -> only 192 CTAs for the logits GEMM).
template <int kBM>
__global__ void __launch_bounds__(kBM * 4)
sgemm_epi_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                 float* __restrict__ C, int ldc, int M, int N, int K,
                 const float* __restrict__ bias, const float* __restrict__ scale,
                 const float* __restrict__ shift, int relu, int k_chunk) {
  // split-K: blockIdx.z owns k in [z*k_chunk, (z+1)*k_chunk) and writes its partial product to C + z*M*ldc (the caller
  // passes bias/scale = nullptr then and finishes with splitk_reduce_kernel); k_chunk >= K means no split.
  constexpr int kThreads = kBM * 4;
  const int k_lo = blockIdx.z * k_chunk;
  const int k_hi = min(K, k_lo + k_chunk);
  C += static_cast<size_t>(blockIdx.z) * M * ldc;
  __shared__ float s_a[kGemmBK][kBM + 4];
  __shared__ float s_b[kGemmBK][kGemmBN + 4];
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * kGemmBN;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = k_lo; k0 < k_hi; k0 += kGemmBK) {
    {   // A tile: kBM rows x 16 k  (thread -> row = tid/4, 4 consecutive k)
      const int r = threadIdx.x >> 2, kk = (threadIdx.x & 3) * 4;
      const int gm = m0 + r;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int gk = k0 + kk + i;
        s_a[kk + i][r] = (gm < M && gk < k_hi) ? A[static_cast<size_t>(gm) * lda + gk] : 0.f;
      }
    }
    // B tile: 16 k x 64 cols, 4 consecutive cols per slot
    for (int slot = threadIdx.x; slot < kGemmBK * kGemmBN / 4; slot += kThreads) {
      const int kk = slot >> 4, c = (slot & 15) * 4;
      const int gk = k0 + kk;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int gn = n0 + c + i;
        s_b[kk][c + i] = (gk < k_hi && gn < N) ? B[static_cast<size_t>(gk) * ldb + gn] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGemmBK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = s_a[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = s_b[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[gn];
      if (scale) v = v * scale[gn] + shift[gn];
      if (relu) v = fmaxf(v, 0.f);
      C[static_cast<size_t>(gm) * ldc + gn] = v;
    }
  }
}

// C[m][n] = ((P0 + P1) + P2) + ... over `parts` split-K partials, added in fixed order (deterministic)
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ partials, float* __restrict__ C, int M, int ldc, int N, int parts) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t total = static_cast<size_t>(M) * ldc;
  if (i >= total || static_cast<int>(i % ldc) >= N) return;
  float v = partials[i];
  for (int z = 1; z < parts; ++z) v += partials[static_cast<size_t>(z) * total + i];
  C[i] = v;
}

// Dense epilogue after the tensor-core GEMM (logits_tc_kernel): C[m][n] = epi(sum of the split-K partials in fixed order),
// epi: v += bias[n]; v = v * scale[n] + shift[n] (Keras BatchNormalization, inference form); relu.  Also writes the value's
// two TF32 halves (low 13 mantissa bits clear) when the result is the A operand of the next tensor-core GEMM, and, when E is set,
// the value once more into the caller's embedding rows (E already points at the step's first row; the index is 64-bit).
__global__ void __launch_bounds__(256)
splitk_reduce_epi_kernel(const float* __restrict__ partials, float* __restrict__ C, float* __restrict__ C_hi, float* __restrict__ C_lo,
                         float* __restrict__ E, int M, int N, int parts, const float* __restrict__ bias, const float* __restrict__ scale,
                         const float* __restrict__ shift, int relu) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t total = static_cast<size_t>(M) * N;
  if (i >= total) return;
  const int n = static_cast<int>(i % N);
  float v = partials[i];
  for (int z = 1; z < parts; ++z) v += partials[static_cast<size_t>(z) * total + i];
  v += bias[n];
  v = v * scale[n] + shift[n];
  if (relu) v = fmaxf(v, 0.f);
  C[i] = v;
  if (E) E[i] = v;
  if (C_hi) {
    const float hi = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
    C_hi[i] = hi;
    C_lo[i] = __uint_as_float(__float_as_uint(v - hi) & 0xffffe000u);
  }
}

// Dense(512 -> 3) + softmax: one warp per window.
__global__ void __launch_bounds__(256)
dense3_softmax_kernel(const float* __restrict__ h2,    // [n][512]
                      const float* __restrict__ Wd,    // [512][3]
                      const float* __restrict__ bd,    // [3]
                      float* __restrict__ probs,       // [n][3]
                      int n) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const float* x = h2 + static_cast<size_t>(w) * kHidden;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int k = lane; k < kHidden; k += 32) {
    const float v = x[k];
    a0 = fmaf(v, Wd[k * 3 + 0], a0);
    a1 = fmaf(v, Wd[k * 3 + 1], a1);
    a2 = fmaf(v, Wd[k * 3 + 2], a2);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    a0 += __shfl_xor_sync(0xffffffffu, a0, off);
    a1 += __shfl_xor_sync(0xffffffffu, a1, off);
    a2 += __shfl_xor_sync(0xffffffffu, a2, off);
  }
  if (lane == 0) {
    a0 += bd[0]; a1 += bd[1]; a2 += bd[2];
    const float m = fmaxf(a0, fmaxf(a1, a2));
    const float e0 = expf(a0 - m), e1 = expf(a1 - m), e2 = expf(a2 - m);
    const float inv = 1.f / (e0 + e1 + e2);
    probs[static_cast<size_t>(w) * 3 + 0] = e0 * inv;
    probs[static_cast<size_t>(w) * 3 + 1] = e1 * inv;
    probs[static_cast<size_t>(w) * 3 + 2] = e2 * inv;
  }
}

// Per-contig reduction: one thread per contig walks its window range in order (fp32 running sum,
// the order tf.math.segment_mean's CPU kernel uses), so the result does not depend on the launch shape.
template <bool kMean>
__global__ void segment_reduce_kernel(const float* __restrict__ probs, const int32_t* __restrict__ offsets,
                                      int n_contigs, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_contigs) return;
  const int b = offsets[c], e = offsets[c + 1];
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  for (int i = b; i < e; ++i) {
    s0 += probs[static_cast<size_t>(i) * 3 + 0];
    s1 += probs[static_cast<size_t>(i) * 3 + 1];
    s2 += probs[static_cast<size_t>(i) * 3 + 2];
  }
  const float cnt = static_cast<float>(e - b);
  if (kMean) {
    const float d = cnt > 0.f ? cnt : 1.f;
    out[static_cast<size_t>(c) * 3 + 0] = s0 / d;
    out[static_cast<size_t>(c) * 3 + 1] = s1 / d;
    out[static_cast<size_t>(c) * 3 + 2] = s2 / d;
  } else {
    out[static_cast<size_t>(c) * 4 + 0] = s0;
    out[static_cast<size_t>(c) * 4 + 1] = s1;
    out[static_cast<size_t>(c) * 4 + 2] = s2;
    out[static_cast<size_t>(c) * 4 + 3] = cnt;
  }
}

// Per-segment sums of 512-wide rows (window embeddings -> per-contig sums): one CTA per segment, 128 threads x 4 columns, so
// each 2 KB row is one fully coalesced 16-byte-per-thread load.  Every column is a plain fp32 running sum in row order (no FMA,
// no tree: the rule of segment_reduce_kernel), so splitting the rows into calls and chaining them through the carry gives the
// same bits as one call.  Segment 0 starts from carry_in when it is set; carry_out is written by the caller (see api.cu).
constexpr int kSegRowThreads = kHidden / 4;
__global__ void __launch_bounds__(kSegRowThreads)
segment_sum_rows_kernel(const float* __restrict__ rows, const int32_t* __restrict__ offsets, const float* __restrict__ carry_in,
                        float* __restrict__ sums) {
  const int c = blockIdx.x;
  const int col = threadIdx.x * 4;
  const int b = offsets[c], e = offsets[c + 1];
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c == 0 && carry_in) s = *reinterpret_cast<const float4*>(carry_in + col);
  for (int i = b; i < e; ++i) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(rows + static_cast<size_t>(i) * kHidden + col));
    s.x = __fadd_rn(s.x, v.x); s.y = __fadd_rn(s.y, v.y); s.z = __fadd_rn(s.z, v.z); s.w = __fadd_rn(s.w, v.w);
  }
  *reinterpret_cast<float4*>(sums + static_cast<size_t>(c) * kHidden + col) = s;
}

}  // namespace gnm
