// Classifier heads with other classes on the frozen encoder: inference (C-class softmax, C-column segment reductions) and
// training of Dense(512) + BatchNormalization + ReLU + Dropout(0.2) + Dense(C, softmax), the stack of the reference's
// create_classifier (genomad/neural_network/model.py:34-45).  The GEMMs are sgemm_epi_kernel / logits_tc_kernel (dense.cuh,
// logits_tc.cuh); this file holds the per-row and per-column kernels around them.  Every reduction runs in a fixed order
// without atomics, so a training run is bitwise reproducible on one device model.
#pragma once
#include "common.cuh"

namespace gnm {

constexpr int kHeadMaxClasses = 32;
constexpr float kHeadDropKeep = 0.8f;                   // Dropout(0.2): kept values are scaled by 1 / 0.8
constexpr uint32_t kHeadDropThreshold = 858993460u;     // ceil(0.2 * 2^32): keep iff hash >= threshold
constexpr int kHeadColBlock = 32;                       // columns per CTA of the column-statistics kernels
constexpr int kHeadRowGroups = 16;                      // row groups per CTA (partials combined in group order)

// lowbias32, as genomad_b200/synth.py's _mix32
__host__ __device__ __forceinline__ uint32_t head_mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}
__host__ __device__ __forceinline__ uint32_t head_key(uint64_t seed) {
  return static_cast<uint32_t>(seed * 0x9E3779B1ull + 0x7F4A7C15ull);
}
// Dropout keep bit of (step, row in the batch, column) for the key of the trainer's seed.
__device__ __forceinline__ bool head_keep(uint32_t key, uint32_t step, uint32_t row, uint32_t col) {
  return head_mix32(head_mix32(head_mix32(key ^ step) + row) + col) >= kHeadDropThreshold;
}

// Rows of fp32 values -> their two TF32 halves, the bits splitk_reduce_epi_kernel writes for the next tensor-core GEMM.
__global__ void __launch_bounds__(256)
head_split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, size_t total) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float v = x[i];
  const float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
  hi[i] = h;
  lo[i] = __uint_as_float(__float_as_uint(v - h) & 0xffffe000u);
}

// Dense(512 -> C) + softmax, one warp per row: the k order, shuffle tree and max / exp / sum / multiply sequence of
// dense3_softmax_kernel, so C = 3 gives its bits.
__global__ void __launch_bounds__(256)
head_softmax_kernel(const float* __restrict__ h2, const float* __restrict__ Wd, const float* __restrict__ bd,
                    float* __restrict__ probs, int n, int C) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const float* x = h2 + static_cast<size_t>(w) * kHidden;
  float a[kHeadMaxClasses];
#pragma unroll
  for (int c = 0; c < kHeadMaxClasses; ++c) a[c] = 0.f;
  for (int k = lane; k < kHidden; k += 32) {
    const float v = x[k];
#pragma unroll
    for (int c = 0; c < kHeadMaxClasses; ++c)
      if (c < C) a[c] = fmaf(v, Wd[k * C + c], a[c]);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1)
#pragma unroll
    for (int c = 0; c < kHeadMaxClasses; ++c)
      if (c < C) a[c] += __shfl_xor_sync(0xffffffffu, a[c], off);
  if (lane == 0) {
    float m = -INFINITY;
#pragma unroll
    for (int c = 0; c < kHeadMaxClasses; ++c)
      if (c < C) { a[c] += bd[c]; m = fmaxf(m, a[c]); }
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < kHeadMaxClasses; ++c)
      if (c < C) { a[c] = expf(a[c] - m); s = c == 0 ? a[c] : s + a[c]; }
    const float inv = 1.f / s;
    float* out = probs + static_cast<size_t>(w) * C;
#pragma unroll
    for (int c = 0; c < kHeadMaxClasses; ++c)
      if (c < C) out[c] = a[c] * inv;
  }
}

// segment_reduce_kernel for C columns: one thread per contig, an fp32 running sum in window order per column.
// kMean: out [n_contigs][C] = sum / max(count, 1); else out [n_contigs][C + 1] = (sums, count).
template <bool kMean>
__global__ void head_segment_reduce_kernel(const float* __restrict__ probs, const int32_t* __restrict__ offsets, int n_contigs,
                                           int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_contigs) return;
  const int b = offsets[c], e = offsets[c + 1];
  const float cnt = static_cast<float>(e - b);
  const float d = cnt > 0.f ? cnt : 1.f;
  const int ld = kMean ? C : C + 1;
  for (int j = 0; j < C; ++j) {
    float s = 0.f;
    for (int i = b; i < e; ++i) s += probs[static_cast<size_t>(i) * C + j];
    out[static_cast<size_t>(c) * ld + j] = kMean ? s / d : s;
  }
  if (!kMean) out[static_cast<size_t>(c) * ld + C] = cnt;
}

// ------------------------------------------------------------------------------------------------------------ training
// Bits of the trainer's input flag (mapped host memory): a batch index outside [0, n_rows), a label outside [0, C).  The
// offending row is read as row 0, the label as class 0, so nothing is read out of bounds; the next call fails.
constexpr int kHeadBadIndex = 1, kHeadBadLabel = 2;

// Batch rows X[idx[r]] -> Xb [B][512] (A of z1 = Xb W1) and XbT [512][B] (A of dW1 = Xb^T dZ1).
__global__ void __launch_bounds__(256)
head_gather_kernel(const float* __restrict__ X, int64_t n_rows, const int64_t* __restrict__ idx, int B, float* __restrict__ Xb,
                   float* __restrict__ XbT, volatile int* bad) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<size_t>(B) * kHidden) return;
  const int r = static_cast<int>(i / kHidden), k = static_cast<int>(i % kHidden);
  int64_t row = idx[r];
  if (row < 0 || row >= n_rows) {
    if (k == 0) *bad |= kHeadBadIndex;
    row = 0;
  }
  const float v = X[static_cast<size_t>(row) * kHidden + k];
  Xb[i] = v;
  XbT[static_cast<size_t>(k) * B + r] = v;
}

// Fixed-order column sum over the CTA's row groups: thread (g, j) sums rows g, g + G, g + 2G, ... in order; group partials are
// then added in group order by the g = 0 thread.  Returns the total on the g = 0 threads.
__device__ __forceinline__ double head_col_total(double part, double (*s)[kHeadColBlock], int g, int j) {
  s[g][j] = part;
  __syncthreads();
  double t = 0.0;
  if (g == 0)
    for (int q = 0; q < kHeadRowGroups; ++q) t += s[q][j];
  __syncthreads();
  return t;
}

// BatchNormalization in training mode + ReLU + dropout, and the moving-statistics update.  CTA = 32 columns x 16 row groups.
//   mu, var (biased) over the batch in fp64, fixed order; inv = 1 / sqrt(var + 1e-3)
//   y = gamma * ((z - mu) * inv) + beta;  h = relu(y) * keep / 0.8
//   moving_mean = 0.99 moving_mean + 0.01 mu;  moving_var = 0.99 moving_var + 0.01 var
// Writes h [B][512], hT [512][B], the keep mask [B][512] and (mu, inv, var) per column.
__global__ void __launch_bounds__(kHeadColBlock * kHeadRowGroups)
head_bn_forward_kernel(const float* __restrict__ z, int B, const float* __restrict__ gamma, const float* __restrict__ beta,
                       float* __restrict__ mov_mean, float* __restrict__ mov_var, uint32_t key, uint32_t step,
                       float* __restrict__ h, float* __restrict__ hT, uint8_t* __restrict__ mask, float* __restrict__ stats) {
  __shared__ double s[kHeadRowGroups][kHeadColBlock];
  __shared__ float s_mu[kHeadColBlock], s_inv[kHeadColBlock];
  const int j = threadIdx.x % kHeadColBlock, g = threadIdx.x / kHeadColBlock;
  const int col = blockIdx.x * kHeadColBlock + j;
  double p = 0.0;
  for (int r = g; r < B; r += kHeadRowGroups) p += z[static_cast<size_t>(r) * kHidden + col];
  const double mu = head_col_total(p, s, g, j) / B;
  if (g == 0) s_mu[j] = static_cast<float>(mu);
  __syncthreads();
  const double mu_all = s_mu[j];
  p = 0.0;
  for (int r = g; r < B; r += kHeadRowGroups) {
    const double d = z[static_cast<size_t>(r) * kHidden + col] - mu_all;
    p += d * d;
  }
  const double var = head_col_total(p, s, g, j) / B;
  if (g == 0) {
    s_inv[j] = static_cast<float>(1.0 / sqrt(var + 1e-3));
    stats[col] = s_mu[j];
    stats[kHidden + col] = s_inv[j];
    stats[2 * kHidden + col] = static_cast<float>(var);
    mov_mean[col] = 0.99f * mov_mean[col] + 0.01f * s_mu[j];
    mov_var[col] = 0.99f * mov_var[col] + 0.01f * static_cast<float>(var);
  }
  __syncthreads();
  const float m = s_mu[j], inv = s_inv[j], ga = gamma[col], be = beta[col];
  for (int r = g; r < B; r += kHeadRowGroups) {
    const size_t i = static_cast<size_t>(r) * kHidden + col;
    const float y = ga * ((z[i] - m) * inv) + be;
    const bool keep = head_keep(key, step, r, col);
    const float v = keep ? fmaxf(y, 0.f) / kHeadDropKeep : 0.f;
    h[i] = v;
    hT[static_cast<size_t>(col) * B + r] = v;
    mask[i] = keep;
  }
}

// Softmax, class-weighted cross-entropy and dZ2 = w_y (p - onehot(y)) / B of one row per warp (lane c = class c); the row's
// loss w_y * (-log softmax(logits)_y) goes to row_loss[r].  With e_c = exp(l_c - max) and a the lowest lane holding the max
// (e_a = 1), both are taken from sums that leave a term out, so neither cancels once the row is classified confidently
// (values just below 1.0f are 2^-24 apart, so 1 - p_y and log(s) would keep only a few bits):
//   s = 1 + sum_{c != a} e_c;  dZ2_y = -w (sum_{c != y} e_c) / s / B;  loss = w ((max - l_y) + log1p(sum_{c != a} e_c)).
__global__ void __launch_bounds__(256)
head_softmax_xent_kernel(const float* __restrict__ logits, int64_t n_rows, const int64_t* __restrict__ idx,
                         const int32_t* __restrict__ labels, const float* __restrict__ class_w, int B, int C,
                         float* __restrict__ dz2, float* __restrict__ row_loss, volatile int* bad) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= B) return;
  const float l = lane < C ? logits[static_cast<size_t>(r) * C + lane] : -INFINITY;
  float m = l;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  const float e = lane < C ? expf(l - m) : 0.f;
  const int a = __ffs(__ballot_sync(0xffffffffu, lane < C && l == m)) - 1;
  const int64_t row = idx[r];
  int y = (row >= 0 && row < n_rows) ? labels[row] : 0;       // a bad index is flagged by head_gather_kernel
  if (y < 0 || y >= C) {
    if (lane == 0) *bad |= kHeadBadLabel;
    y = 0;
  }
  float sa = lane == a ? 0.f : e, sy = lane == y ? 0.f : e;   // sums over c != a and over c != y
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    sa += __shfl_xor_sync(0xffffffffu, sa, off);
    sy += __shfl_xor_sync(0xffffffffu, sy, off);
  }
  const float s = 1.f + sa;
  const float w = class_w[y];
  if (lane < C) dz2[static_cast<size_t>(r) * C + lane] = w * (lane == y ? -(sy / s) : e / s) / static_cast<float>(B);
  const float ly = __shfl_sync(0xffffffffu, l, y);
  if (lane == 0) row_loss[r] = w * ((m - ly) + log1pf(sa));
}

// One CTA of 64 threads: loss = sum_r row_loss[r] / B, db2[c] = sum_r dZ2[r][c], in row order (fp64).
__global__ void __launch_bounds__(64)
head_loss_db2_kernel(const float* __restrict__ row_loss, const float* __restrict__ dz2, int B, int C, float* __restrict__ loss,
                     float* __restrict__ db2) {
  const int t = threadIdx.x;
  if (t < C) {
    double s = 0.0;
    for (int r = 0; r < B; ++r) s += dz2[static_cast<size_t>(r) * C + t];
    db2[t] = static_cast<float>(s);
  } else if (t == kHeadMaxClasses) {
    double s = 0.0;
    for (int r = 0; r < B; ++r) s += row_loss[r];
    *loss = static_cast<float>(s / B);
  }
}

// W2 [512][C] -> W2T [C][512] (B operand of dH = dZ2 W2^T)
__global__ void __launch_bounds__(256)
head_transpose_w2_kernel(const float* __restrict__ W2, int C, float* __restrict__ W2T) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kHidden * C) return;
  const int k = i / C, c = i % C;
  W2T[static_cast<size_t>(c) * kHidden + k] = W2[i];
}

// Backward of BatchNormalization (training mode) + ReLU + dropout, CTA = 32 columns x 16 row groups (fp64 column sums, fixed
// order).  With xh = (z - mu) inv, y = gamma xh + beta, dy = dH * keep / 0.8 * (y > 0):
//   dbeta = sum dy;  dgamma = sum dy xh;  dz = gamma inv (dy - dbeta / B - xh dgamma / B);  db1 = sum dz.
__global__ void __launch_bounds__(kHeadColBlock * kHeadRowGroups)
head_bn_backward_kernel(const float* __restrict__ z, const float* __restrict__ dH, const uint8_t* __restrict__ mask, int B,
                        const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ stats,
                        float* __restrict__ dz, float* __restrict__ db1, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ double s[kHeadRowGroups][kHeadColBlock];
  __shared__ float s_db[kHeadColBlock], s_dg[kHeadColBlock];
  const int j = threadIdx.x % kHeadColBlock, g = threadIdx.x / kHeadColBlock;
  const int col = blockIdx.x * kHeadColBlock + j;
  const float m = stats[col], inv = stats[kHidden + col], ga = gamma[col], be = beta[col];
  double pb = 0.0, pg = 0.0;
  for (int r = g; r < B; r += kHeadRowGroups) {
    const size_t i = static_cast<size_t>(r) * kHidden + col;
    const float xh = (z[i] - m) * inv;
    const float y = ga * xh + be;
    const float dy = (mask[i] && y > 0.f) ? dH[i] / kHeadDropKeep : 0.f;
    pb += dy;
    pg += static_cast<double>(dy) * xh;
  }
  const double db = head_col_total(pb, s, g, j);
  const double dg = head_col_total(pg, s, g, j);
  if (g == 0) {
    s_db[j] = static_cast<float>(db); s_dg[j] = static_cast<float>(dg);
    dbeta[col] = s_db[j]; dgamma[col] = s_dg[j];
  }
  __syncthreads();
  const float mb = s_db[j] / B, mg = s_dg[j] / B, gi = ga * inv;
  double pz = 0.0;
  for (int r = g; r < B; r += kHeadRowGroups) {
    const size_t i = static_cast<size_t>(r) * kHidden + col;
    const float xh = (z[i] - m) * inv;
    const float y = ga * xh + be;
    const float dy = (mask[i] && y > 0.f) ? dH[i] / kHeadDropKeep : 0.f;
    const float v = gi * (dy - mb - xh * mg);
    dz[i] = v;
    pz += v;
  }
  const double d1 = head_col_total(pz, s, g, j);
  if (g == 0) db1[col] = static_cast<float>(d1);
}

// Adam (Keras 3): m += (g - m)(1 - b1); v += (g^2 - v)(1 - b2); p -= (m * alpha) / (sqrt(v) + eps),
// alpha = lr sqrt(1 - b2^t) / (1 - b1^t).  alpha, 1 - b1 and 1 - b2 come from the host, computed in double and rounded once
// (as Keras does: 1 - 0.999f in fp32 would be off by 1.3e-5 relative).
__global__ void __launch_bounds__(256)
head_adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, size_t n,
                 float alpha, float one_m_b1, float one_m_b2, float eps) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i];
  const float mi = m[i] + (gi - m[i]) * one_m_b1;
  const float vi = v[i] + (gi * gi - v[i]) * one_m_b2;
  m[i] = mi;
  v[i] = vi;
  p[i] -= (mi * alpha) / (sqrtf(vi) + eps);
}

}  // namespace gnm
