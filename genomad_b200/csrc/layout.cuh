// Embedding map: a UMAP layout (McInnes, Healy & Melville 2018) of the rows of an embeddings file on two axes, computed as
// umap-learn computes it except where DESIGN.md, "Embedding map" says otherwise.  Spec: include/gnm.h.  Every reduction runs in
// a fixed order without atomics, so a map is bitwise reproducible for the same rows, k, epochs and seed.
#pragma once
#include "common.cuh"
#include "head.cuh"
#include "novelty.cuh"

namespace gnm {

constexpr int kMpMaxK = 64;
constexpr int kMpBisect = 64;                         // umap-learn's smooth_knn_dist: 64 bisection steps,
constexpr double kMpTolerance = 1e-5;                 //   an early exit at |sum - target| < 1e-5,
constexpr double kMpMinScale = 1e-3;                  //   and a floor of 1e-3 x the mean distance
constexpr int kMpMeanThreads = 1024;
constexpr int kMpEigThreads = kHidden;             // one thread per row of S
constexpr int kMpEigIters = 512;                      // subspace steps: the top-2 subspace error falls as (l3 / l2)^steps
constexpr int kMpNegatives = 5;
constexpr float kMpA = 1.57694346f;                   // 1 / (1 + a x^2b) fitted to min_dist = 0.1, spread = 1
constexpr float kMpB = 0.89506088f;
constexpr float kMpClip = 4.0f;
constexpr double kMpNoise = 1e-4 / 2147483648.0;      // noise = (h - 2^31 + 0.5) * kMpNoise, in (-1e-4, 1e-4)

__device__ __forceinline__ double mp_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);   // the same bits in every lane
  return v;
}
__device__ __forceinline__ float mp_warp_sumf(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- memberships
// *mean_d = the mean of d = 1 - s over all n k entries: thread t sums rows t, t + 1024, ... in row and list order, then the
// 1024 partials are added in a fixed tree.  One CTA.
__global__ void __launch_bounds__(kMpMeanThreads)
mp_mean_kernel(const float* __restrict__ sim, int n, int k, double* __restrict__ mean_d) {
  __shared__ double part[kMpMeanThreads];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kMpMeanThreads)
    for (int p = 0; p < k; ++p) s += 1.0 - static_cast<double>(sim[static_cast<size_t>(i) * k + p]);
  part[threadIdx.x] = s;
  __syncthreads();
  for (int h = kMpMeanThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) *mean_d = part[0] / (static_cast<double>(n) * k);
}

// One warp per row i, entries p = lane and lane + 32: rho_i, sigma_i by umap-learn's bisection for
// sum_p f(d_ip - rho_i) = log2(k + 1), f(x) = exp(-x / sigma) for x > 0 and 1 otherwise, then w_ip = f(d_ip - rho_i).
__global__ void __launch_bounds__(256)
mp_sigma_kernel(const float* __restrict__ sim, int n, int k, const double* __restrict__ mean_d, double* __restrict__ rho,
                double* __restrict__ sigma, double* __restrict__ w) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const float* s = sim + static_cast<size_t>(i) * k;
  const bool h0 = lane < k, h1 = lane + 32 < k;
  const double d0 = h0 ? 1.0 - static_cast<double>(s[lane]) : 0.0;
  const double d1 = h1 ? 1.0 - static_cast<double>(s[lane + 32]) : 0.0;
  double m = INFINITY;
  if (h0 && d0 > 0.0) m = d0;
  if (h1 && d1 > 0.0) m = fmin(m, d1);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
  const double r = m == INFINITY ? 0.0 : m;
  const double target = log2(static_cast<double>(k) + 1.0);
  double lo = 0.0, hi = INFINITY, mid = 1.0;
  for (int it = 0; it < kMpBisect; ++it) {
    double ps = 0.0;
    if (h0) ps += d0 - r > 0.0 ? exp(-((d0 - r) / mid)) : 1.0;
    if (h1) ps += d1 - r > 0.0 ? exp(-((d1 - r) / mid)) : 1.0;
    ps = mp_warp_sum(ps);                             // every lane takes the same branch
    if (fabs(ps - target) < kMpTolerance) break;
    if (ps > target) {
      hi = mid;
      mid = (lo + hi) / 2.0;
    } else {
      lo = mid;
      mid = hi == INFINITY ? mid * 2.0 : (lo + hi) / 2.0;
    }
  }
  const double row_mean = mp_warp_sum(d0 + d1) / k;
  const double floor_ = kMpMinScale * (r > 0.0 ? row_mean : *mean_d);
  const double sg = mid < floor_ ? floor_ : mid;
  double* wr = w + static_cast<size_t>(i) * k;
  if (h0) wr[lane] = d0 - r > 0.0 ? exp(-((d0 - r) / sg)) : 1.0;
  if (h1) wr[lane + 32] = d1 - r > 0.0 ? exp(-((d1 - r) / sg)) : 1.0;
  if (lane == 0) { rho[i] = r; sigma[i] = sg; }
}

// One thread per directed entry (i, p), j = idx[i][p]: b = w_jq if i = idx[j][q], else 0, and the fuzzy union a + b - a b.  The
// unordered pair is emitted once, from the lower index when the entries are mutual, else from the row that holds it; an entry
// that does not emit gets -1.  A separate kernel from mp_sigma_kernel because it reads w of other rows.
__global__ void __launch_bounds__(256)
mp_union_kernel(const long long* __restrict__ idx, const double* __restrict__ w, int n, int k, double* __restrict__ uni) {
  const long long e = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (e >= static_cast<long long>(n) * k) return;
  const long long i = e / k, j = idx[e];
  if (j < 0 || j >= n) { uni[e] = -1.0; return; }                  // padding: no edge
  const long long* lj = idx + j * k;
  int q = -1;
  for (int t = 0; t < k; ++t)
    if (lj[t] == i) { q = t; break; }
  const double a = w[e], b = q >= 0 ? w[j * k + q] : 0.0;
  uni[e] = (q < 0 || i < j) ? a + b - a * b : -1.0;
}

// ---- PCA initialisation
// x^ = x / |x|, the norm and the quotient in fp64, stored fp32; a zero row stays zero.  One warp per row.
__global__ void __launch_bounds__(256)
mp_normalize_kernel(const float* __restrict__ x, int n, float* __restrict__ xh) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const float* r = x + static_cast<size_t>(i) * kHidden;
  double v[kHidden / 32], ss = 0.0;
#pragma unroll
  for (int q = 0; q < kHidden / 32; ++q) {
    v[q] = static_cast<double>(r[lane + 32 * q]);
    ss = fma(v[q], v[q], ss);
  }
  const double nrm = sqrt(mp_warp_sum(ss));
  float* o = xh + static_cast<size_t>(i) * kHidden;
#pragma unroll
  for (int q = 0; q < kHidden / 32; ++q) o[lane + 32 * q] = nrm > 0.0 ? static_cast<float>(v[q] / nrm) : 0.f;
}

// The novelty fit's covariance kernels at C = 1 read fit row r as (idx[r], labels[idx[r]]): every row, label 0.
__global__ void __launch_bounds__(256) mp_iota_kernel(int n, long long* __restrict__ idx, int* __restrict__ labels) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) { idx[i] = i; labels[i] = 0; }
}

// Sum of v[0..511] over the CTA, in a fixed tree; every thread gets it.  red: kMpEigThreads doubles.
__device__ __forceinline__ double mp_block_dot(const double* a, const double* b, double* red) {
  const int t = threadIdx.x;
  red[t] = a[t] * b[t];
  __syncthreads();
  for (int h = kMpEigThreads / 2; h > 0; h >>= 1) {
    if (t < h) red[t] += red[t + h];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// Top-2 eigenvectors of the symmetric S [512][512] (fp64): subspace iteration from a fixed hashed start, kMpEigIters steps of
// V <- orth(S V) by Gram-Schmidt, then a Rayleigh-Ritz rotation of the 2 x 2 projection, and each vector's sign set so that its
// largest-magnitude component (the first one on ties) is positive.  A direction S maps to 0 keeps its previous vector (S = 0:
// the start).  One CTA; V [2][512].
__global__ void __launch_bounds__(kMpEigThreads)
mp_eig_kernel(const double* __restrict__ S, double* __restrict__ V) {
  __shared__ double v[2][kHidden], u[2][kHidden], red[kMpEigThreads];
  __shared__ int s_arg[kMpEigThreads];
  const int t = threadIdx.x;
  for (int c = 0; c < 2; ++c) v[c][t] = static_cast<double>(head_mix32(head_mix32(0x5EEDu + c) + t)) / 4294967296.0 - 0.5;
  __syncthreads();
  auto orth = [&](double (*src)[kHidden]) {          // v <- Gram-Schmidt(src), keeping v where a norm is 0
    const double n1 = sqrt(mp_block_dot(src[0], src[0], red));
    if (n1 > 0.0) v[0][t] = src[0][t] / n1;
    __syncthreads();
    const double d = mp_block_dot(v[0], src[1], red);
    src[1][t] -= d * v[0][t];
    __syncthreads();
    const double n2 = sqrt(mp_block_dot(src[1], src[1], red));
    if (n2 > 0.0) {
      v[1][t] = src[1][t] / n2;
    } else {                                          // keep v2, made orthogonal to the new v1
      const double d2 = mp_block_dot(v[0], v[1], red);
      v[1][t] -= d2 * v[0][t];
      __syncthreads();
      const double n3 = sqrt(mp_block_dot(v[1], v[1], red));
      if (n3 > 0.0) v[1][t] /= n3;
    }
    __syncthreads();
  };
  auto apply = [&]() {                                // u = S v, k ascending
    const double* row = S + static_cast<size_t>(t) * kHidden;
    double s0 = 0.0, s1 = 0.0;
    for (int q = 0; q < kHidden; ++q) {
      const double sq = row[q];
      s0 = fma(sq, v[0][q], s0);
      s1 = fma(sq, v[1][q], s1);
    }
    u[0][t] = s0;
    u[1][t] = s1;
    __syncthreads();
  };
  for (int q = 0; q < 2; ++q) u[q][t] = v[q][t];
  __syncthreads();
  orth(u);
  for (int it = 0; it < kMpEigIters; ++it) {
    apply();
    orth(u);
  }
  apply();
  const double h11 = mp_block_dot(v[0], u[0], red), h12 = mp_block_dot(v[0], u[1], red), h22 = mp_block_dot(v[1], u[1], red);
  // one Jacobi rotation diagonalises the 2 x 2 projection (Numerical Recipes' t, c, s); the larger Ritz value goes first
  double cs = 1.0, sn = 0.0, l1 = h11, l2 = h22;
  if (h12 != 0.0) {
    const double th = (h22 - h11) / (2.0 * h12);
    const double tn = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
    cs = 1.0 / sqrt(tn * tn + 1.0);
    sn = tn * cs;
    l1 = h11 - tn * h12;
    l2 = h22 + tn * h12;
  }
  {
    const double a = v[0][t], b = v[1][t];
    const double w1 = cs * a - sn * b, w2 = sn * a + cs * b;
    u[0][t] = l1 >= l2 ? w1 : w2;
    u[1][t] = l1 >= l2 ? w2 : w1;
  }
  __syncthreads();
  for (int q = 0; q < 2; ++q) {
    red[t] = fabs(u[q][t]);
    s_arg[t] = t;
    __syncthreads();
    for (int h = kMpEigThreads / 2; h > 0; h >>= 1) {
      if (t < h && (red[t + h] > red[t] || (red[t + h] == red[t] && s_arg[t + h] < s_arg[t]))) {
        red[t] = red[t + h];
        s_arg[t] = s_arg[t + h];
      }
      __syncthreads();
    }
    const bool neg = u[q][s_arg[0]] < 0.0;
    V[q * kHidden + t] = neg ? -u[q][t] : u[q][t];
    __syncthreads();
  }
}

// proj [n][2] (fp64) = (x^ - center) . v_c, one warp per row, columns lane + 32 q, then the warp tree.
__global__ void __launch_bounds__(256)
mp_project_kernel(const float* __restrict__ xh, int n, const double* __restrict__ center, const double* __restrict__ V,
                  double* __restrict__ proj) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const float* x = xh + static_cast<size_t>(i) * kHidden;
  double p0 = 0.0, p1 = 0.0;
#pragma unroll 4
  for (int q = 0; q < kHidden / 32; ++q) {
    const int j = lane + 32 * q;
    const double d = static_cast<double>(x[j]) - center[j];
    p0 = fma(d, V[j], p0);
    p1 = fma(d, V[kHidden + j], p1);
  }
  p0 = mp_warp_sum(p0);
  p1 = mp_warp_sum(p1);
  if (lane == 0) { proj[2 * static_cast<size_t>(i)] = p0; proj[2 * static_cast<size_t>(i) + 1] = p1; }
}

// One CTA: out[0] = max |v[e]| over e < m; with `axes`, out[0..1] = the per-axis minimum and out[2..3] the maximum of the
// float pairs y [m][2] instead.  Minima and maxima do not depend on the order.
__global__ void __launch_bounds__(1024)
mp_extent_kernel(const double* __restrict__ v, const float* __restrict__ y, long long m, double* __restrict__ out) {
  __shared__ double red[4][1024];
  const int t = threadIdx.x;
  double a[4] = {0.0, INFINITY, INFINITY, -INFINITY};
  if (v) {
    for (long long e = t; e < m; e += 1024) a[0] = fmax(a[0], fabs(v[e]));
  } else {
    a[0] = INFINITY;
    a[3] = -INFINITY;
    a[2] = -INFINITY;
    for (long long e = t; e < m; e += 1024) {
      a[0] = fmin(a[0], static_cast<double>(y[2 * e]));
      a[1] = fmin(a[1], static_cast<double>(y[2 * e + 1]));
      a[2] = fmax(a[2], static_cast<double>(y[2 * e]));
      a[3] = fmax(a[3], static_cast<double>(y[2 * e + 1]));
    }
  }
  for (int q = 0; q < 4; ++q) red[q][t] = a[q];
  __syncthreads();
  for (int h = 512; h > 0; h >>= 1) {
    if (t < h) {
      if (v) {
        red[0][t] = fmax(red[0][t], red[0][t + h]);
      } else {
        red[0][t] = fmin(red[0][t], red[0][t + h]);
        red[1][t] = fmin(red[1][t], red[1][t + h]);
        red[2][t] = fmax(red[2][t], red[2][t + h]);
        red[3][t] = fmax(red[3][t], red[3][t + h]);
      }
    }
    __syncthreads();
  }
  if (t < (v ? 1 : 4)) out[t] = red[t][0];
}

// y [n][2] = fp32(proj * 10 / max|proj|) + noise (proj alone skipped when max|proj| = 0), noise the fp32 value of
// (mix32(mix32(key ^ row) + axis) - 2^31 + 0.5) * 1e-4 / 2^31, exact in fp64 but for the one product.
__global__ void __launch_bounds__(256)
mp_noise_kernel(const double* __restrict__ proj, int n, const double* __restrict__ amax, uint32_t key, float* __restrict__ y) {
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= 2 * n) return;
  const uint32_t h = head_mix32(head_mix32(key ^ static_cast<uint32_t>(e >> 1)) + static_cast<uint32_t>(e & 1));
  const float noise = static_cast<float>((static_cast<double>(h) - 2147483647.5) * kMpNoise);
  const double m = *amax;
  const float base = m > 0.0 ? static_cast<float>(proj[e] * (10.0 / m)) : 0.f;
  y[e] = __fadd_rn(base, noise);
}

// y = 10 (y - min) / (max - min) per axis in fp32, as umap-learn rescales its initialisation (an axis of one value becomes 0).
__global__ void __launch_bounds__(256) mp_rescale_kernel(float* __restrict__ y, int n, const double* __restrict__ ext) {
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= 2 * n) return;
  const float lo = static_cast<float>(ext[e & 1]), hi = static_cast<float>(ext[2 + (e & 1)]);
  const float range = __fsub_rn(hi, lo);
  y[e] = range > 0.f ? __fdiv_rn(__fmul_rn(10.f, __fsub_rn(y[e], lo)), range) : 0.f;
}

// ---- layout epochs
// Edge with epochs-per-sample eps is sampled at epoch e >= 1 iff floor(e / eps) > floor((e - 1) / eps), in fp64.
__device__ __forceinline__ bool mp_sampled(double eps, int e) {
  return floor(static_cast<double>(e) / eps) > floor(static_cast<double>(e - 1) / eps);
}
__device__ __forceinline__ float mp_clip(float v) { return fminf(fmaxf(v, -kMpClip), kMpClip); }

// One synchronous epoch e >= 1: Yn[i] = Y[i] + alpha * (sum of the forces on i), one warp per vertex over its CSR row.  Lane l
// takes the row's entries l, l + 32, ... in order; for a sampled entry (i, j) at CSR position p it adds the attraction twice
// (umap-learn samples both directed entries, and both move i) and the repulsion of the 5 negatives
// mix32(mix32(ekey + p) + s) mod n, s = 0..4, skipping i, where ekey = mix32(key ^ e).  The lanes' sums meet in the
// xor tree.  No atomics: the epoch's bits depend only on its inputs.
__global__ void __launch_bounds__(256)
mp_epoch_kernel(const long long* __restrict__ row_ptr, const int* __restrict__ col, const double* __restrict__ eps, int n, int e,
                uint32_t ekey, float alpha, const float2* __restrict__ Y, float2* __restrict__ Yn) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const float2 yi = Y[i];
  float fx = 0.f, fy = 0.f;
  const long long end = row_ptr[i + 1];
  for (long long p = row_ptr[i] + lane; p < end; p += 32) {
    if (!mp_sampled(eps[p], e)) continue;
    const float2 yj = Y[col[p]];
    float dx = yi.x - yj.x, dy = yi.y - yj.y;
    float d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
    if (d2 > 0.f) {
      const float gc = __fdiv_rn(__fmul_rn(-2.f * kMpA * kMpB, powf(d2, kMpB - 1.f)), __fadd_rn(__fmul_rn(kMpA, powf(d2, kMpB)), 1.f));
      fx = __fadd_rn(fx, 2.f * mp_clip(__fmul_rn(gc, dx)));
      fy = __fadd_rn(fy, 2.f * mp_clip(__fmul_rn(gc, dy)));
    }
    const uint32_t hp = head_mix32(ekey + static_cast<uint32_t>(p));
#pragma unroll
    for (int s = 0; s < kMpNegatives; ++s) {
      const int kk = static_cast<int>(head_mix32(hp + s) % static_cast<uint32_t>(n));
      if (kk == i) continue;
      const float2 yk = Y[kk];
      dx = yi.x - yk.x;
      dy = yi.y - yk.y;
      d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
      if (d2 > 0.f) {
        const float gc = __fdiv_rn(2.f * kMpB, __fmul_rn(__fadd_rn(0.001f, d2), __fadd_rn(__fmul_rn(kMpA, powf(d2, kMpB)), 1.f)));
        fx = __fadd_rn(fx, mp_clip(__fmul_rn(gc, dx)));
        fy = __fadd_rn(fy, mp_clip(__fmul_rn(gc, dy)));
      }
    }
  }
  fx = mp_warp_sumf(fx);
  fy = mp_warp_sumf(fy);
  if (lane == 0) Yn[i] = make_float2(__fadd_rn(yi.x, __fmul_rn(alpha, fx)), __fadd_rn(yi.y, __fmul_rn(alpha, fy)));
}

}  // namespace gnm
