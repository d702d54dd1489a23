// Window regions (gnm_window_regions, include/gnm.h): an HMM decode of each sequence's window-score profile into class regions.
//
//   wr_decode_kernel  one warp per sequence, lane k = class k (C <= 32), kWrWarps warps per CTA.  Four passes over the
//                     sequence's windows, each in tiles of 32 windows whose raw rows are loaded into registers a tile ahead:
//     forward         scaled forward recursion in the linear domain (alpha-hat to the workspace) and, in the same steps, the
//                     Viterbi recursion in the log domain; the emission factors exp(eps) and log-emissions eps of a tile, and
//                     its per-window transition constants, are staged in shared memory before its steps, so no exp / log sits
//                     on the recursions' chains.  The traceback data of a window is (argmax, second argmax) of the previous
//                     column and the ballot of the lanes that stay: 6 bytes whatever C is.
//     backward        scaled backward recursion; gamma = alpha-hat * beta-hat / sum overwrites alpha-hat (fp64) and goes out as
//                     the fp32 posterior.
//     traceback       from the lowest-index argmax of the last column, 32 steps per tile from shuffled traceback data.
//     regions         each run of equal states, in window order: fp64 sums of gamma(class) and of every class's score, written
//                     at the row of the run's first window with its coordinates; every row gets its run-start flag.
// Nothing depends on another sequence, so a sequence's results are bitwise the same in any call, order or chunk.
// DESIGN.md, "Window regions".
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gnm {

constexpr int kWrTile = 32;                      // windows per tile
constexpr int kWrWarps = 4;                      // warps (sequences) per CTA
constexpr int kWrMaxClasses = 32;
constexpr int kWrSmemPerWarp = 2 * kWrTile * kWrMaxClasses * 8 + kWrTile * 4 * 8;
constexpr int kWrSmem = kWrWarps * kWrSmemPerWarp;

struct WrParams {
  const float* scores;          // [W][C]
  const int32_t* offsets;       // [n_seqs + 1]; window index = offsets[i] - offsets[0]
  const int64_t* start;         // [W]
  const int32_t* length;        // [W]
  int n_seqs, C;
  long long stride;
  double tau, log1p_mq, inv_c, log_c;   // s / 6000, log1p(-rho C / (C - 1)), 1 / C, ln C
  float* posterior;             // [W][C]
  int32_t* state;               // [W]
  uint8_t* first;               // [W]
  int64_t* r_start;             // [W] (rows of run starts)
  int64_t* r_end;
  int32_t* r_windows;
  float* r_posterior;
  float* r_scores;              // [W][C]
  double* gam;                  // workspace [W][C]: alpha-hat, then gamma
  uint32_t* bp_mask;            // workspace [W]
  uint16_t* bp_idx;             // workspace [W]
};

__device__ __forceinline__ double wr_sum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double wr_max(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// raw inputs of one tile: lane k holds the scores of class k, lane j the start of window j and of the window before it
struct WrRaw {
  float p[kWrTile];
  long long a, ap;
};

__device__ __forceinline__ void wr_load(const WrParams& P, int w0, int nt, int b, int lane, WrRaw& r) {
#pragma unroll
  for (int j = 0; j < kWrTile; ++j)
    r.p[j] = (j < nt && lane < P.C) ? __ldg(P.scores + static_cast<size_t>(w0 + j) * P.C + lane) : 1.f;
  r.a = lane < nt ? __ldg(P.start + w0 + lane) : 0;
  r.ap = (lane < nt && w0 + lane > b) ? __ldg(P.start + w0 + lane - 1) : r.a;
}

// Stage a tile: E[j][k] = exp(eps), L[j][k] = eps (-inf for lanes >= C), K[j] = (lambda^g, O_g, ln T_g, ln O_g) with
// O_g = (1 - lambda^g) / C and T_g = 1 - (C - 1) O_g, computed without cancellation through expm1 / log1p.
__device__ __forceinline__ void wr_stage(const WrParams& P, const WrRaw& r, int nt, int lane, double* E, double* L, double* K) {
#pragma unroll
  for (int j = 0; j < kWrTile; ++j) {
    if (j < nt) {
      const double eps = P.tau * log(fmax(static_cast<double>(r.p[j]), 1e-30));
      E[j * kWrMaxClasses + lane] = lane < P.C ? exp(eps) : 0.0;
      L[j * kWrMaxClasses + lane] = lane < P.C ? eps : -INFINITY;
    }
  }
  if (lane < nt) {
    const long long gap = r.a > r.ap ? (r.a - r.ap) / P.stride : 1;   // the first window of a sequence: unused
    const double x = static_cast<double>(gap) * P.log1p_mq;
    const double o = -expm1(x) * P.inv_c;
    K[4 * lane + 0] = exp(x);
    K[4 * lane + 1] = o;
    K[4 * lane + 2] = log1p(-(P.C - 1) * o);
    K[4 * lane + 3] = log(o);
  }
}

__global__ void __launch_bounds__(kWrWarps * 32)
wr_decode_kernel(const WrParams P) {
  extern __shared__ __align__(16) uint8_t wr_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int seq = blockIdx.x * kWrWarps + warp;
  if (seq >= P.n_seqs) return;
  double* E = reinterpret_cast<double*>(wr_smem + warp * kWrSmemPerWarp);
  double* L = E + kWrTile * kWrMaxClasses;
  double* K = L + kWrTile * kWrMaxClasses;
  const int base = __ldg(P.offsets);
  const int b = __ldg(P.offsets + seq) - base, e = __ldg(P.offsets + seq + 1) - base;
  const int n = e - b;
  if (n <= 0) return;
  const int C = P.C, ntiles = (n + kWrTile - 1) / kWrTile;
  const bool act = lane < C;
  WrRaw raw;

  // ---------------------------------------------------------------- forward + Viterbi
  double ah = 0.0, dl = -INFINITY, m1 = 0.0, m2 = 0.0;
  int a1 = 0, a2 = 0;
  wr_load(P, b, min(kWrTile, n), b, lane, raw);
  for (int t = 0; t < ntiles; ++t) {
    const int w0 = b + t * kWrTile, nt = min(kWrTile, e - w0);
    wr_stage(P, raw, nt, lane, E, L, K);
    __syncwarp();
    if (t + 1 < ntiles) wr_load(P, w0 + kWrTile, min(kWrTile, e - w0 - kWrTile), b, lane, raw);
#pragma unroll 2
    for (int j = 0; j < nt; ++j) {
      const int w = w0 + j;
      const double ex = E[j * kWrMaxClasses + lane], ep = L[j * kWrMaxClasses + lane];
      double at;
      if (w == b) {
        at = ex;
        dl = ep - P.log_c;
      } else {
        const double lam = K[4 * j], o = K[4 * j + 1], lt = K[4 * j + 2], lo = K[4 * j + 3];
        at = ex * fma(lam, ah, o);
        const double stay = dl + lt, move = (lane == a1 ? m2 : m1) + lo;
        const bool st = stay >= move;
        dl = ep + (st ? stay : move);
        const uint32_t mask = __ballot_sync(0xffffffffu, st);
        if (lane == 0) {
          P.bp_mask[w] = mask;
          P.bp_idx[w] = static_cast<uint16_t>(a1 | (a2 << 8));
        }
      }
      ah = at / wr_sum(at);
      if (act) P.gam[static_cast<size_t>(w) * C + lane] = ah;
      m1 = wr_max(dl);
      a1 = __ffs(__ballot_sync(0xffffffffu, dl == m1)) - 1;
      m2 = wr_max(lane == a1 ? -INFINITY : dl);
      a2 = __ffs(__ballot_sync(0xffffffffu, lane != a1 && dl == m2)) - 1;
    }
    __syncwarp();
  }
  const int last_state = a1;

  // ---------------------------------------------------------------- backward, posteriors
  double bh = act ? 1.0 : 0.0;
  {
    const int t = ntiles - 1, w0 = b + t * kWrTile;
    wr_load(P, w0, e - w0, b, lane, raw);
  }
  for (int t = ntiles - 1; t >= 0; --t) {
    const int w0 = b + t * kWrTile, nt = min(kWrTile, e - w0);
    wr_stage(P, raw, nt, lane, E, L, K);
    __syncwarp();
    if (t > 0) wr_load(P, w0 - kWrTile, kWrTile, b, lane, raw);
#pragma unroll 2
    for (int j = nt - 1; j >= 0; --j) {
      const int w = w0 + j;
      const size_t g = static_cast<size_t>(w) * C + lane;
      const double al = act ? P.gam[g] : 0.0;
      const double u = E[j * kWrMaxClasses + lane] * bh;
      const double z = al * bh;
      const double gm = z / wr_sum(z);
      if (act) {
        P.gam[g] = gm;
        P.posterior[g] = static_cast<float>(gm);
      }
      if (w > b) bh = fma(K[4 * j], u / wr_sum(u), K[4 * j + 1]);
    }
    __syncwarp();
  }

  // ---------------------------------------------------------------- traceback
  int s = last_state;
  for (int t = ntiles - 1; t >= 0; --t) {
    const int w0 = b + t * kWrTile, nt = min(kWrTile, e - w0);
    const uint32_t mk = lane < nt && w0 + lane > b ? P.bp_mask[w0 + lane] : 0u;
    const uint32_t ix = lane < nt && w0 + lane > b ? P.bp_idx[w0 + lane] : 0u;
    int mine = 0;
#pragma unroll
    for (int j = kWrTile - 1; j >= 0; --j) {
      const uint32_t mj = __shfl_sync(0xffffffffu, mk, j), ij = __shfl_sync(0xffffffffu, ix, j);
      if (j < nt) {
        if (lane == j) mine = s;
        if (w0 + j > b) {
          const int x1 = static_cast<int>(ij & 255u), x2 = static_cast<int>(ij >> 8);
          s = (mj >> s) & 1u ? s : (s != x1 ? x1 : x2);
        }
      }
    }
    if (lane < nt) P.state[w0 + lane] = mine;
  }
  __syncwarp();

  // ---------------------------------------------------------------- regions
  double sp = 0.0, sg = 0.0;
  int r0 = b, cnt = 0;
  long long rs = 0;
  for (int t = 0; t < ntiles; ++t) {
    const int w0 = b + t * kWrTile, nt = min(kWrTile, e - w0);
    const int w = w0 + lane;
    int st = 0, stp = -1, stn = -1;
    long long lb = 0, rb = 0;
    if (lane < nt) {
      st = P.state[w];
      const long long a = P.start[w], c = a + P.length[w] / 2;
      if (w > b) {
        stp = P.state[w - 1];
        lb = (P.start[w - 1] + P.length[w - 1] / 2 + c) / 2;
      } else {
        lb = a;
      }
      if (w + 1 < e) {
        stn = P.state[w + 1];
        rb = (c + P.start[w + 1] + P.length[w + 1] / 2) / 2;
      } else {
        rb = a + P.length[w];
      }
      P.first[w] = stp != st;
    }
    const uint32_t firsts = __ballot_sync(0xffffffffu, lane < nt && stp != st);
    const uint32_t lasts = __ballot_sync(0xffffffffu, lane < nt && stn != st);
#pragma unroll 4
    for (int j = 0; j < nt; ++j) {
      const int wj = w0 + j;
      const int sj = __shfl_sync(0xffffffffu, st, j);
      const long long lbj = __shfl_sync(0xffffffffu, lb, j), rbj = __shfl_sync(0xffffffffu, rb, j);
      if ((firsts >> j) & 1u) {
        r0 = wj; rs = lbj; cnt = 0; sp = 0.0; sg = 0.0;
      }
      const size_t g = static_cast<size_t>(wj) * C + lane;
      if (act) {
        sp += static_cast<double>(P.scores[g]);
        if (lane == sj) sg += P.gam[g];
      }
      ++cnt;
      if ((lasts >> j) & 1u) {
        if (act) P.r_scores[static_cast<size_t>(r0) * C + lane] = static_cast<float>(sp / cnt);
        if (lane == sj) P.r_posterior[r0] = static_cast<float>(sg / cnt);
        if (lane == 0) {
          P.r_start[r0] = rs;
          P.r_end[r0] = rbj;
          P.r_windows[r0] = cnt;
        }
      }
    }
  }
}

}  // namespace gnm
