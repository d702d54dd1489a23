// Head novelty: a Gaussian model of the encoder embeddings a head was trained on (one mean per class, one shared covariance),
// fitted and scored in fp64 on the DMMA tensor cores (mma.sync m16n8k16 f64).  Model and semantics: include/gnm.h and
// DESIGN.md, "Head novelty".  Every reduction runs in a fixed order without atomics: a fit is bitwise reproducible for the same
// rows, and a row's distances do not depend on the batch it is scored in.
#pragma once
#include "common.cuh"

namespace gnm {

constexpr int kNvMaxClasses = 32;
constexpr double kNvAlpha = 0.01;                   // shrinkage towards (tr S / 512) I
constexpr int kNvSumRows = 4096;                    // rows per block of the class sums (partials combined in block order)
constexpr int kNvChunk = 8192;                      // rows per K chunk of the scatter GEMM (partials combined in chunk order)
constexpr int kNvTile = 64;                         // output tile of the scatter and score GEMMs
constexpr int kNvTiles = kHidden / kNvTile;         // 8
constexpr int kNvTriTiles = kNvTiles * (kNvTiles + 1) / 2;   // 36 lower-triangular tiles of S
constexpr int kNvK = 16;                            // k per mma.m16n8k16
constexpr int kNvThreads = 128;                     // 4 warps, 2 x 2 over a 64 x 64 tile, 32 x 32 each
constexpr int kNvKM = kNvTile + 4;                  // row stride of the k-major scatter operands (fp64; 2-way banks)
constexpr int kNvMK = kNvK + 4;                     // row stride of the m-major score operands
constexpr int kNvYS = kNvTile + 4;                  // row stride of the score's Y tile
constexpr int kNvFactorThreads = 1024;
// score kernel shared memory: A, B operands, Y tile, per-(row, class) sums, the column tile of the whitened means
constexpr int kNvScoreSmem = (2 * kNvTile * kNvMK + kNvTile * kNvYS + kNvTile * kNvMaxClasses + kNvMaxClasses * kNvTile) * 8;

// Status of a fit, in device memory: the first error found (gnm_novelty_fit names it), the smallest pivot and tr S.
enum { kNvOk = 0, kNvBadIndex = 1, kNvBadLabel = 2, kNvEmptyClass = 3, kNvNoVariation = 4, kNvBadPivot = 5, kNvNonFinite = 6 };
struct NvStatus {
  int code;
  int arg;
  double min_pivot;
  double trace;
};

// D += A B for one m16n8k16 f64 tile.  Fragments (lane = 4 g + t):
//   A a[i] = A[g + 8 (i & 1)][t + 4 (i >> 1)];  B b[i] = B[t + 4 i][g];  D d[i] = D[g + 8 (i >> 1)][2 t + (i & 1)].
__device__ __forceinline__ void nv_mma(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
      "{%12, %13, %14, %15}, {%0, %1, %2, %3};\n"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
        "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// One k16 step of a warp's 32 x 32 block of a 64 x 64 tile: A(m, k) = a_at(m, k), B(k, n) = b_at(k, n) from shared memory.
template <class FA, class FB>
__device__ __forceinline__ void nv_warp_step(double (&acc)[2][4][4], int wm, int wn, int lane, FA a_at, FB b_at) {
  const int g = lane >> 2, t = lane & 3;
  double b[4][4];
#pragma unroll
  for (int ni = 0; ni < 4; ++ni)
#pragma unroll
    for (int i = 0; i < 4; ++i) b[ni][i] = b_at(t + 4 * i, wn * 32 + ni * 8 + g);
#pragma unroll
  for (int mi = 0; mi < 2; ++mi) {
    double a[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = a_at(wm * 32 + mi * 16 + g + 8 * (i & 1), t + 4 * (i >> 1));
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) nv_mma(acc[mi][ni], a, b[ni]);
  }
}

// Fit row r of the fit list -> (row of X, label), or -1 with the error flagged (bad rows are left out of the fit; it fails).
__device__ __forceinline__ int64_t nv_fit_row(const int64_t* __restrict__ idx, const int32_t* __restrict__ labels, int64_t n_rows,
                                              int C, int64_t r, int* y, NvStatus* st) {
  const int64_t row = idx[r];
  if (row < 0 || row >= n_rows) { st->code = kNvBadIndex; return -1; }
  const int c = labels[row];
  if (c < 0 || c >= C) { st->code = kNvBadLabel; return -1; }
  *y = c;
  return row;
}

// Per block of kNvSumRows fit rows: the fp64 sum of each class's rows and the class counts.  Thread j owns column j of every
// class's sum in shared memory and adds the block's rows in order.  part [block][C][512], cnt [block][C].
__global__ void __launch_bounds__(kHidden)
nv_class_sums_kernel(const float* __restrict__ X, int64_t n_rows, const int64_t* __restrict__ idx, const int32_t* __restrict__ labels,
                     int64_t n_fit, int C, double* __restrict__ part, long long* __restrict__ cnt, NvStatus* st) {
  extern __shared__ double nv_sum[];                     // [C][512]
  __shared__ long long s_cnt[kNvMaxClasses];
  const int j = threadIdx.x;
  for (int c = 0; c < C; ++c) nv_sum[c * kHidden + j] = 0.0;
  if (j < kNvMaxClasses) s_cnt[j] = 0;
  __syncthreads();
  const int64_t b = static_cast<int64_t>(blockIdx.x) * kNvSumRows;
  const int64_t e = b + kNvSumRows < n_fit ? b + kNvSumRows : n_fit;
  for (int64_t r = b; r < e; ++r) {
    int y = 0;
    const int64_t row = nv_fit_row(idx, labels, n_rows, C, r, &y, st);
    if (row < 0) continue;
    nv_sum[y * kHidden + j] += static_cast<double>(X[row * kHidden + j]);
    if (j == 0) s_cnt[y]++;
  }
  __syncthreads();
  for (int c = 0; c < C; ++c) part[(static_cast<size_t>(blockIdx.x) * C + c) * kHidden + j] = nv_sum[c * kHidden + j];
  if (j < C) cnt[static_cast<size_t>(blockIdx.x) * C + j] = s_cnt[j];
}

// Block c < C: mu_c = (sum of the block partials in block order) / N_c.  Block C: the center = (sum over classes, in class order,
// of those same class sums) / N.  mu [C][512], center [512], counts [C].
__global__ void __launch_bounds__(kHidden)
nv_means_kernel(const double* __restrict__ part, const long long* __restrict__ cnt, int n_blocks, int C, int64_t n_fit,
                double* __restrict__ mu, double* __restrict__ center, long long* __restrict__ counts, NvStatus* st) {
  const int j = threadIdx.x, c0 = blockIdx.x;
  if (c0 < C) {
    double s = 0.0;
    long long n = 0;
    for (int b = 0; b < n_blocks; ++b) {
      s += part[(static_cast<size_t>(b) * C + c0) * kHidden + j];
      n += cnt[static_cast<size_t>(b) * C + c0];
    }
    if (n == 0) {
      if (j == 0 && st->code == kNvOk) { st->code = kNvEmptyClass; st->arg = c0; }
      mu[static_cast<size_t>(c0) * kHidden + j] = 0.0;
    } else {
      mu[static_cast<size_t>(c0) * kHidden + j] = s / static_cast<double>(n);
    }
    if (j == 0) counts[c0] = n;
  } else {
    double tot = 0.0;
    for (int c = 0; c < C; ++c) {
      double s = 0.0;
      for (int b = 0; b < n_blocks; ++b) s += part[(static_cast<size_t>(b) * C + c) * kHidden + j];
      tot += s;
    }
    center[j] = tot / static_cast<double>(n_fit);
  }
}

// Lower-triangular tile t of the 8 x 8 grid of 64 x 64 tiles -> (row tile, column tile), row tile >= column tile.
__device__ __forceinline__ void nv_tri_tile(int t, int* ta, int* tb) {
  int a = 0;
  while (t > a) { t -= a + 1; ++a; }
  *ta = a; *tb = t;
}

// Partial scatter of one K chunk for one lower tile: sum over the chunk's rows of d d^T, d = x - mu_y centred in fp64 as the
// operands are loaded.  part [chunk][36][64][64].
__global__ void __launch_bounds__(kNvThreads)
nv_scatter_kernel(const float* __restrict__ X, int64_t n_rows, const int64_t* __restrict__ idx, const int32_t* __restrict__ labels,
                  int64_t n_fit, int C, const double* __restrict__ mu, double* __restrict__ part, NvStatus* st) {
  __shared__ double sA[kNvK][kNvKM], sB[kNvK][kNvKM];   // [k = fit row][m or n = column within the tile]
  __shared__ int64_t s_row[kNvK];
  __shared__ int s_lab[kNvK];
  int ta, tb;
  nv_tri_tile(blockIdx.x, &ta, &tb);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wm = warp >> 1, wn = warp & 1;
  const int64_t r_begin = static_cast<int64_t>(blockIdx.y) * kNvChunk;
  const int64_t r_end = r_begin + kNvChunk < n_fit ? r_begin + kNvChunk : n_fit;
  double acc[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mi][ni][i] = 0.0;
  const int col = tid & 63, k_first = tid >> 6;         // each thread loads column `col` of rows k_first, k_first + 2, ...
  for (int64_t r0 = r_begin; r0 < r_end; r0 += kNvK) {
    if (tid < kNvK) {
      int y = 0;
      const int64_t r = r0 + tid;
      const int64_t row = r < r_end ? nv_fit_row(idx, labels, n_rows, C, r, &y, st) : -1;
      s_row[tid] = row;
      s_lab[tid] = y;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kNvK / 2; ++q) {
      const int k = k_first + 2 * q;
      const int64_t row = s_row[k];
      double va = 0.0, vb = 0.0;
      if (row >= 0) {
        const float* x = X + row * kHidden;
        const double* m = mu + static_cast<size_t>(s_lab[k]) * kHidden;
        va = static_cast<double>(x[ta * kNvTile + col]) - m[ta * kNvTile + col];
        vb = static_cast<double>(x[tb * kNvTile + col]) - m[tb * kNvTile + col];
      }
      sA[k][col] = va;
      sB[k][col] = vb;
    }
    __syncthreads();
    nv_warp_step(acc, wm, wn, lane, [&](int m, int k) { return sA[k][m]; }, [&](int k, int n) { return sB[k][n]; });
    __syncthreads();
  }
  double* out = part + (static_cast<size_t>(blockIdx.y) * kNvTriTiles + blockIdx.x) * kNvTile * kNvTile;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i)
        out[(wm * 32 + mi * 16 + g + 8 * (i >> 1)) * kNvTile + wn * 32 + ni * 8 + 2 * t + (i & 1)] = acc[mi][ni][i];
}

// S = (sum of the chunk partials in chunk order) / N, from the lower triangle (row >= column) and mirrored, so S is exactly
// symmetric.  grid (36, 16), 256 threads: one element of a tile per thread.
__global__ void __launch_bounds__(256)
nv_scatter_reduce_kernel(const double* __restrict__ part, int n_chunks, int64_t n_fit, double* __restrict__ S) {
  int ta, tb;
  nv_tri_tile(blockIdx.x, &ta, &tb);
  const int e = blockIdx.y * 256 + threadIdx.x;
  const int m = e / kNvTile, n = e % kNvTile;
  const int i = ta * kNvTile + m, j = tb * kNvTile + n;
  if (i < j) return;
  double s = 0.0;
  for (int c = 0; c < n_chunks; ++c) s += part[(static_cast<size_t>(c) * kNvTriTiles + blockIdx.x) * kNvTile * kNvTile + e];
  s /= static_cast<double>(n_fit);
  S[static_cast<size_t>(i) * kHidden + j] = s;
  S[static_cast<size_t>(j) * kHidden + i] = s;
}

// One CTA: Sigma = (1 - alpha) S + alpha (tr S / 512) I, then its Cholesky factor L (lower; zeros above) in place of Sigma,
// right-looking, column by column.  A non-finite tr S (a fit row with a NaN or an infinity), tr S <= 0 and a pivot that is not
// > 0 stop the fit (NvStatus).
__global__ void __launch_bounds__(kNvFactorThreads)
nv_factor_kernel(const double* __restrict__ S, double* __restrict__ L, NvStatus* st) {
  __shared__ double s_tr;
  const int tid = threadIdx.x;
  if (st->code != kNvOk) return;
  if (tid == 0) {
    double tr = 0.0;
    for (int k = 0; k < kHidden; ++k) tr += S[static_cast<size_t>(k) * (kHidden + 1)];
    s_tr = tr;
    st->trace = tr;
  }
  __syncthreads();
  const double tr = s_tr;
  if (!isfinite(tr) || !(tr > 0.0)) {
    if (tid == 0) st->code = isfinite(tr) ? kNvNoVariation : kNvNonFinite;
    return;
  }
  const double shrink = kNvAlpha * (tr / kHidden);
  for (int e = tid; e < kHidden * kHidden; e += kNvFactorThreads) {
    const int i = e / kHidden, j = e % kHidden;
    L[e] = j <= i ? (1.0 - kNvAlpha) * S[e] + (i == j ? shrink : 0.0) : 0.0;
  }
  __syncthreads();
  double min_pivot = INFINITY;
  const int ty = tid >> 5, tx = tid & 31;
  for (int k = 0; k < kHidden; ++k) {
    const double p = L[static_cast<size_t>(k) * (kHidden + 1)];
    if (!(p > 0.0) || !isfinite(p)) {                     // every thread read the same p: all leave together
      if (tid == 0) { st->code = kNvBadPivot; st->arg = k; }
      return;
    }
    min_pivot = fmin(min_pivot, p);
    const double d = sqrt(p);
    __syncthreads();                                      // every thread has read p
    if (tid == 0) L[static_cast<size_t>(k) * (kHidden + 1)] = d;
    for (int i = k + 1 + tid; i < kHidden; i += kNvFactorThreads) L[static_cast<size_t>(i) * kHidden + k] /= d;
    __syncthreads();
    for (int i = k + 1 + ty; i < kHidden; i += kNvFactorThreads / 32) {
      const double lik = L[static_cast<size_t>(i) * kHidden + k];
      for (int j = k + 1 + tx; j <= i; j += 32)
        L[static_cast<size_t>(i) * kHidden + j] -= lik * L[static_cast<size_t>(j) * kHidden + k];
    }
    __syncthreads();
  }
  if (tid == 0) st->min_pivot = min_pivot;
}

// P = L^-1 (lower triangular), one thread per column j by forward substitution in row order:
//   P[j][j] = 1 / L[j][j];  P[i][j] = -(sum_{k=j}^{i-1} L[i][k] P[k][j]) / L[i][i]  (k ascending).
__global__ void __launch_bounds__(128)
nv_inverse_kernel(const double* __restrict__ L, double* __restrict__ P, const NvStatus* st) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= kHidden || st->code != kNvOk) return;
  for (int i = 0; i < j; ++i) P[static_cast<size_t>(i) * kHidden + j] = 0.0;
  P[static_cast<size_t>(j) * kHidden + j] = 1.0 / L[static_cast<size_t>(j) * (kHidden + 1)];
  for (int i = j + 1; i < kHidden; ++i) {
    double s = 0.0;
    for (int k = j; k < i; ++k) s += L[static_cast<size_t>(i) * kHidden + k] * P[static_cast<size_t>(k) * kHidden + j];
    P[static_cast<size_t>(i) * kHidden + j] = -s / L[static_cast<size_t>(i) * (kHidden + 1)];
  }
}

// m_c = P (mu_c - center): block c, thread i, k ascending over the lower triangle.
__global__ void __launch_bounds__(kHidden)
nv_whiten_means_kernel(const double* __restrict__ P, const double* __restrict__ mu, const double* __restrict__ center,
                       double* __restrict__ m, const NvStatus* st) {
  const int c = blockIdx.x, i = threadIdx.x;
  if (st->code != kNvOk) return;
  double s = 0.0;
  for (int k = 0; k <= i; ++k) s += P[static_cast<size_t>(i) * kHidden + k] * (mu[static_cast<size_t>(c) * kHidden + k] - center[k]);
  m[static_cast<size_t>(c) * kHidden + i] = s;
}

// Column tile ct of Y = (x - center) P^T for the 64 rows from row0 (rows >= n read as 0) into a warp's accumulators: k ascending
// in k16 steps over the tiles up to the diagonal (P is zero above it).  sA, sB: [64][kNvMK] each.  nv_score_kernel and
// nv_residual_kernel share it, so their Y are the same bits.
__device__ __forceinline__ void nv_y_tile(double (&acc)[2][4][4], const float* __restrict__ x, int n, int64_t row0,
                                          const double* __restrict__ center, const double* __restrict__ P, int ct, double* sA,
                                          double* sB, int tid, int wm, int wn, int lane) {
  const int lk = tid & 15, lr = tid >> 4;                // loader: column lk of rows lr, lr + 8, ...
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mi][ni][i] = 0.0;
  const int k_end = (ct + 1) * kNvTile;
  for (int k0 = 0; k0 < k_end; k0 += kNvK) {
    const double cen = center[k0 + lk];
#pragma unroll
    for (int q = 0; q < kNvTile / 8; ++q) {
      const int r = lr + 8 * q;
      const int64_t gr = row0 + r;
      sA[r * kNvMK + lk] = gr < n ? static_cast<double>(x[gr * kHidden + k0 + lk]) - cen : 0.0;
      sB[r * kNvMK + lk] = P[static_cast<size_t>(ct * kNvTile + r) * kHidden + k0 + lk];
    }
    __syncthreads();
    nv_warp_step(acc, wm, wn, lane, [&](int m, int k) { return sA[m * kNvMK + k]; },
                 [&](int k, int nn) { return sB[nn * kNvMK + k]; });
    __syncthreads();
  }
}

// D [n][C] (fp32) = || P (x - center) - m_c ||^2 / 512 per row, computed in fp64: per 64-row block, the column tiles of
// Y = (x - center) P^T in order (k tiles above the diagonal, where P is zero, skipped), each followed by the epilogue that adds
// sum_j (Y[r][j] - m_c[j])^2 over the tile's columns in column order into the (row, class) sum in shared memory.  A row's
// arithmetic is the same whatever block, position or n it is scored in.
__global__ void __launch_bounds__(kNvThreads)
nv_score_kernel(const float* __restrict__ x, int n, const double* __restrict__ center, const double* __restrict__ P,
                const double* __restrict__ means, int C, float* __restrict__ out) {
  extern __shared__ double nv_smem[];
  double* sA = nv_smem;                                  // [64 rows][kNvMK]: x - center
  double* sB = sA + kNvTile * kNvMK;                     // [64 columns of Y][kNvMK]: P rows
  double* sY = sB + kNvTile * kNvMK;                     // [64][kNvYS]
  double* sD = sY + kNvTile * kNvYS;                     // [64][32]: (row, class) sums
  double* sM = sD + kNvTile * kNvMaxClasses;             // [C][64]: the tile's columns of m_c
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wm = warp >> 1, wn = warp & 1;
  const int64_t row0 = static_cast<int64_t>(blockIdx.x) * kNvTile;
  for (int p = tid; p < kNvTile * kNvMaxClasses; p += kNvThreads) sD[p] = 0.0;
  for (int ct = 0; ct < kNvTiles; ++ct) {
    double acc[2][4][4];
    nv_y_tile(acc, x, n, row0, center, P, ct, sA, sB, tid, wm, wn, lane);
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int i = 0; i < 4; ++i)
          sY[(wm * 32 + mi * 16 + g + 8 * (i >> 1)) * kNvYS + wn * 32 + ni * 8 + 2 * t + (i & 1)] = acc[mi][ni][i];
    for (int p = tid; p < C * kNvTile; p += kNvThreads)
      sM[p] = means[static_cast<size_t>(p / kNvTile) * kHidden + ct * kNvTile + p % kNvTile];
    __syncthreads();
    for (int p = tid; p < kNvTile * C; p += kNvThreads) {
      const int r = p / C, c = p % C;
      double s = sD[r * kNvMaxClasses + c];
      for (int jj = 0; jj < kNvTile; ++jj) {
        const double d = sY[r * kNvYS + jj] - sM[c * kNvTile + jj];
        s = fma(d, d, s);
      }
      sD[r * kNvMaxClasses + c] = s;
    }
    __syncthreads();
  }
  for (int p = tid; p < kNvTile * C; p += kNvThreads) {
    const int r = p / C, c = p % C;
    const int64_t gr = row0 + r;
    if (gr < n) out[gr * C + c] = static_cast<float>(sD[r * kNvMaxClasses + c] / kHidden);
  }
}

// ---- gradient of a window's distance to its target class (novelty attributions; DESIGN.md, "Head novelty")
// r [n][512] (fp64) = P (x - center) - m_c, c = target[row]: nv_score_kernel's Y, and r[j] the same bits as the difference its
// epilogue squares, stored straight from the accumulators.
__global__ void __launch_bounds__(kNvThreads)
nv_residual_kernel(const float* __restrict__ x, int n, const double* __restrict__ center, const double* __restrict__ P,
                   const double* __restrict__ means, const int32_t* __restrict__ target, double* __restrict__ r) {
  __shared__ double sA[kNvTile * kNvMK], sB[kNvTile * kNvMK];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wm = warp >> 1, wn = warp & 1, g = lane >> 2, t = lane & 3;
  const int64_t row0 = static_cast<int64_t>(blockIdx.x) * kNvTile;
  for (int ct = 0; ct < kNvTiles; ++ct) {
    double acc[2][4][4];
    nv_y_tile(acc, x, n, row0, center, P, ct, sA, sB, tid, wm, wn, lane);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int i = 0; i < 4; i += 2) {
        const int64_t gr = row0 + wm * 32 + mi * 16 + g + 8 * (i >> 1);
        if (gr >= n) continue;
        const double* m = means + static_cast<size_t>(target[gr]) * kHidden + ct * kNvTile;
        double* out = r + gr * kHidden + ct * kNvTile;
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          const int j = wn * 32 + ni * 8 + 2 * t;
          out[j] = acc[mi][ni][i] - m[j];
          out[j + 1] = acc[mi][ni][i + 1] - m[j + 1];
        }
      }
  }
}

// g [n][512] (fp32) = dD_c / dx = (2 / 512) P^T r, computed in fp64 and rounded once: block (64 rows, column tile cj),
// g[j] = sum_{i >= j} r[i] P[i][j] over the k tiles from the diagonal down (P is zero above it), k ascending in k16 steps.
__global__ void __launch_bounds__(kNvThreads)
nv_grad_kernel(const double* __restrict__ r, int n, const double* __restrict__ P, float* __restrict__ g_out) {
  __shared__ double sA[kNvTile * kNvMK], sB[kNvTile * kNvMK];   // [64 rows][k], [64 columns of g][k]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wm = warp >> 1, wn = warp & 1;
  const int64_t row0 = static_cast<int64_t>(blockIdx.x) * kNvTile;
  const int cj = blockIdx.y;
  double acc[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mi][ni][i] = 0.0;
  const int lk = tid & 15, lr = tid >> 4;                // A loader: column lk of rows lr, lr + 8, ...
  const int bn = tid & 63, bk = tid >> 6;                // B loader: column bn of P rows k0 + bk, k0 + bk + 2, ...
  for (int k0 = cj * kNvTile; k0 < kHidden; k0 += kNvK) {
#pragma unroll
    for (int q = 0; q < kNvTile / 8; ++q) {
      const int m = lr + 8 * q;
      const int64_t gr = row0 + m;
      sA[m * kNvMK + lk] = gr < n ? r[gr * kHidden + k0 + lk] : 0.0;
      const int k = bk + 2 * q;
      sB[bn * kNvMK + k] = P[static_cast<size_t>(k0 + k) * kHidden + cj * kNvTile + bn];
    }
    __syncthreads();
    nv_warp_step(acc, wm, wn, lane, [&](int m, int k) { return sA[m * kNvMK + k]; },
                 [&](int k, int nn) { return sB[nn * kNvMK + k]; });
    __syncthreads();
  }
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t gr = row0 + wm * 32 + mi * 16 + g + 8 * (i >> 1);
        if (gr < n)
          g_out[gr * kHidden + cj * kNvTile + wn * 32 + ni * 8 + 2 * t + (i & 1)] =
              static_cast<float>(acc[mi][ni][i] * (2.0 / kHidden));
      }
}

// out[2 i] = dist[i][target[i * t_stride]] (row 0 for every i when `broadcast`): a window's distance to its own target, from
// its distance row (t_stride = the rows per window of the target list) or from the baseline's one row.
__global__ void __launch_bounds__(256)
nv_pick_kernel(const float* __restrict__ dist, int broadcast, int n, int C, const int32_t* __restrict__ target, int t_stride,
               float* __restrict__ out) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  out[static_cast<size_t>(i) * 2] = dist[(broadcast ? 0 : static_cast<size_t>(i) * C) + target[static_cast<size_t>(i) * t_stride]];
}

}  // namespace gnm
