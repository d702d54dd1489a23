// Nearest neighbours in the encoder's embedding space (gnm_embedding_neighbours, include/gnm.h): for every query row, the k
// reference rows of highest cosine similarity, under the total order (similarity descending, reference index ascending).
//
//   nb_prep_kernel      one warp per 512-wide row: the row prescaled by the power of two that brings its max |x| into [1, 2), the
//                       fp32 norm (each lane sums its 16 squares in order, then a fixed xor butterfly), x / norm (a zero norm
//                       gives the zero row), and the TF32 halves of split_tf32 (logits_tc.cuh)
//                       as two row-major [n][512] fp32 matrices that TMA reads as 128-byte-swizzled K-major tiles.
//   nb_search_kernel    the similarity tile S = Q R^T of 128 queries x 192 references on the tensor cores with the recipe of
//                       logits_tc_kernel (D = Qhi Rhi + Qlo Rhi + Qhi Rlo per K = 8 step, K chunks of 32 in ascending order, one
//                       fp32 accumulator, no split-K), and the top-k taken from the accumulator registers: each query row keeps
//                       its k best in shared memory together with the current worst entry (the admission threshold) in the
//                       registers of the quad of lanes that holds the row's fragments.  A fragment value below the threshold
//                       costs one compare and one vote; only survivors go through the exact (similarity, index) comparison and
//                       replace the worst entry.  S never leaves the registers.  A CTA owns one query tile and a contiguous range
//                       of reference tiles (a split), and writes its lists sorted to the workspace.
//   nb_finalize_kernel  one warp per query: merges the splits' lists in split order and writes global int64 indices.
//   nb_merge_kernel     one warp per query: merges a second set of lists into the first, in place (gnm_neighbours_merge).
//
// Every similarity is computed by the same instruction sequence over the same operand bits whatever tile, split, call or rank
// computes it, and the lists are merged under a total order on distinct keys, so the result is bitwise independent of how the
// reference set is partitioned.  DESIGN.md, "Embedding neighbours".
#pragma once
#include <cuda.h>
#include <math_constants.h>
#include <climits>
#include "common.cuh"
#include "logits_tc.cuh"

namespace gnm {

constexpr int kNbDim = 512;
constexpr int kNbBM = 128, kNbBN = 192, kNbBK = 32;              // queries x references x fp32 K per chunk (128 B per row)
constexpr int kNbChunks = kNbDim / kNbBK;                          // 16
constexpr int kNbStages = 2;
constexpr int kNbATile = kNbBM * 128, kNbBTile = kNbBN * 128;      // 16 KB, 24 KB
constexpr int kNbStageBytes = 2 * kNbATile + 2 * kNbBTile;          // Q hi | Q lo | R hi | R lo = 80 KB
constexpr int kNbMaxK = 64;
constexpr int kNbThreads = 384;                                     // warp 0: TMA; warpgroups 1, 2: MMA + top-k, 64 queries each
constexpr int kNbMinSplits = 8;   // reference splits per query tile at least (when there are that many reference tiles): the
                                  // CTAs resident at once then cover ~16 query tiles, whose Q operands stay in L2
constexpr int kNbRowMax = (1 << 30);                                // row counts: 32-bit offsets inside the kernels
__host__ __device__ constexpr int nb_smem_bytes(int k) { return kNbStages * kNbStageBytes + kNbBM * k * 8 + 1024 + 64; }

struct NbSearchParams {
  float* part_sim;          // [splits][n_query][k], each list sorted
  int32_t* part_idx;        // reference rows of this call, -1 = empty
  int n_query, n_ref, k;
  int splits;               // CTA b: split b % splits of query tile b / splits
  int tiles_per_split;      // reference tiles of kNbBN rows per split
  long long self_off;       // query q never returns reference row q + self_off (LLONG_MIN: no exclusion)
  DeviceStatus* status;
};

// the total order: a ranks before b
__device__ __forceinline__ bool nb_beats(float as, long long ai, float bs, long long bi) {
  return as > bs || (as == bs && ai < bi);
}

// 2^e as a float, exactly, for e in [-149, 127]
__device__ __forceinline__ float nb_pow2(int e) {
  return e >= -126 ? __int_as_float((e + 127) << 23) : __int_as_float(1 << (e + 149));
}

// Prescale: the row is first multiplied by the power of two 2^-E that brings its max |x| into [1, 2) (one exact factor, or two
// for a subnormal max, which needs more than 2^127), so the fp32 sum of squares neither overflows (a row with sum x^2 > FLT_MAX
// would get norm inf and become the zero row) nor loses digits to subnormal squares.  The product is exact whenever the scaled
// entry is a normal float, so:
//   * when every partial sum of squares is a normal float (or zero) both before and after the prescale -- e.g. every nonzero
//     x_i^2 is normal, scaled or not, and sum x^2 is finite -- the halves are bitwise those of the same recipe without it (the
//     fma, sqrt and division results are those unscaled times exact powers of two, and x / norm is the same quotient);
//   * x * 2^e gives bitwise the halves of x whenever every nonzero entry of x and of x * 2^e is a normal float (both prescale to
//     the same row).
__global__ void __launch_bounds__(256) nb_prep_kernel(const float* __restrict__ x, int n, float* __restrict__ hi,
                                                      float* __restrict__ lo) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n) return;
  const float4* src = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * kNbDim);
  float4 v[4];
  float mx = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[i] = src[lane + 32 * i];
    mx = fmaxf(mx, fmaxf(fmaxf(fabsf(v[i].x), fabsf(v[i].y)), fmaxf(fabsf(v[i].z), fabsf(v[i].w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  const int E = mx > 0.f ? ilogbf(mx) : 0;                                        // mx * 2^-E in [1, 2)
  const float f0 = E < -127 ? nb_pow2(64) : 1.f, f1 = nb_pow2(E < -127 ? -E - 64 : -E);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[i].x = v[i].x * f0 * f1; v[i].y = v[i].y * f0 * f1; v[i].z = v[i].z * f0 * f1; v[i].w = v[i].w * f0 * f1;
    ss = fmaf(v[i].x, v[i].x, ss); ss = fmaf(v[i].y, v[i].y, ss); ss = fmaf(v[i].z, v[i].z, ss); ss = fmaf(v[i].w, v[i].w, ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);     // a + b == b + a: every lane gets the same bits
  const float nrm = sqrtf(ss);
  float4* dh = reinterpret_cast<float4*>(hi + static_cast<size_t>(row) * kNbDim);
  float4* dl = reinterpret_cast<float4*>(lo + static_cast<size_t>(row) * kNbDim);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float y[4] = {v[i].x, v[i].y, v[i].z, v[i].w}, h[4], l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) split_tf32(nrm > 0.f ? y[e] / nrm : 0.f, h[e], l[e]);
    dh[lane + 32 * i] = make_float4(h[0], h[1], h[2], h[3]);
    dl[lane + 32 * i] = make_float4(l[0], l[1], l[2], l[3]);
  }
}

// The quad (4 lanes) that holds query row `rowl` offers the 4 candidates (one per lane) of one fragment position, in lane
// order.  ws / wi / wp: the row's worst list entry (similarity, row, slot), the same in the quad's 4 lanes.  Warp-uniform.
__device__ __forceinline__ void nb_offer(float v, int col, int rowl, int self_col, int n_ref, int k, float& ws, int& wi, int& wp,
                                         float* lsim, int* lidx) {
  const int lane = threadIdx.x & 31;
  const unsigned want = __ballot_sync(0xffffffffu, v >= ws);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int src = (lane & ~3) | q;
    const float cv = __shfl_sync(0xffffffffu, v, src);
    const int cc = __shfl_sync(0xffffffffu, col, src);
    const bool ok = ((want >> src) & 1u) && cc < n_ref && cc != self_col && nb_beats(cv, cc, ws, wi);
    if (!__any_sync(0xffffffffu, ok)) continue;
    if (ok && (lane & 3) == 0) { lsim[rowl * k + wp] = cv; lidx[rowl * k + wp] = cc; }
    __syncwarp();
    // new worst: lowest similarity, then highest row, then highest slot (a total order, so the quad agrees)
    float bs = CUDART_INF_F; int bi = 0x7fffffff, bp = -1;
    if (ok) {
      for (int p = lane & 3; p < k; p += 4) {
        const float xs = lsim[rowl * k + p]; const int xi = lidx[rowl * k + p];
        if (xs < bs || (xs == bs && (xi > bi || (xi == bi && p > bp)))) { bs = xs; bi = xi; bp = p; }
      }
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float os = __shfl_xor_sync(0xffffffffu, bs, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o), op = __shfl_xor_sync(0xffffffffu, bp, o);
      if (os < bs || (os == bs && (oi > bi || (oi == bi && op > bp)))) { bs = os; bi = oi; bp = op; }
    }
    if (ok) { ws = bs; wi = bi; wp = bp; }
    __syncwarp();
  }
}

// The mainloop shared by nb_search_kernel and nb_mask_kernel (clusters.cuh), so that a pair's similarity has the same bits in
// both: the same TMA ring, the same wgmma sequence over the same operand bits.  A CTA of kNbThreads: warp 0 lane 0 produces,
// warpgroups 1 and 2 consume; the ring is smem[0, kNbStages * kNbStageBytes) with barriers full / empty.
__device__ __forceinline__ void nb_ring_init(const CUtensorMap* tm_q_hi, const CUtensorMap* tm_q_lo, const CUtensorMap* tm_r_hi,
                                             const CUtensorMap* tm_r_lo, uint64_t* full, uint64_t* empty) {
  tma_prefetch_desc(tm_q_hi); tma_prefetch_desc(tm_q_lo); tma_prefetch_desc(tm_r_hi); tma_prefetch_desc(tm_r_lo);
  for (int i = 0; i < kNbStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
  fence_barrier_init();
}

// TMA producer: query tile m0 against reference tiles t0 .. t0 + nt - 1, K chunks ascending.
__device__ __forceinline__ void nb_produce(const CUtensorMap* tm_q_hi, const CUtensorMap* tm_q_lo, const CUtensorMap* tm_r_hi,
                                           const CUtensorMap* tm_r_lo, uint8_t* smem, uint64_t* full, uint64_t* empty, int m0,
                                           int t0, int nt, DeviceStatus* status) {
  const uint64_t pol = l2_policy_evict_last();       // Q is re-read for every reference tile, R by every resident query tile
  for (int it = 0; it < nt * kNbChunks; ++it) {
    const int s = it % kNbStages;
    const uint32_t ph = (it / kNbStages) & 1;
    mbar_wait(&empty[s], ph ^ 1, status, 700 + s);
    mbar_arrive_expect_tx(&full[s], kNbStageBytes);
    uint8_t* st = smem + s * kNbStageBytes;
    const int k0 = (it % kNbChunks) * kNbBK, r0 = (t0 + it / kNbChunks) * kNbBN;
    tma_load_2d_hint(st, tm_q_hi, &full[s], k0, m0, pol);
    tma_load_2d_hint(st + kNbATile, tm_q_lo, &full[s], k0, m0, pol);
    tma_load_2d_hint(st + 2 * kNbATile, tm_r_hi, &full[s], k0, r0, pol);
    tma_load_2d_hint(st + 2 * kNbATile + kNbBTile, tm_r_lo, &full[s], k0, r0, pol);
  }
}

// Consumer warpgroup g: the tile tt of its run, S = Qhi Rhi + Qlo Rhi + Qhi Rlo per K = 8 step, K chunks ascending, into d
// (register i holds row 8 ((i >> 1) & 1) + lane / 4 of the warp's 16, column 8 (i >> 2) + 2 (lane % 4) + (i & 1); wgmma.cuh).
__device__ __forceinline__ void nb_tile_mma(float (&d)[96], uint32_t base, uint64_t* full, uint64_t* empty, int g, int tt,
                                            DeviceStatus* status) {
  const int lane = threadIdx.x & 31;
  for (int c = 0; c < kNbChunks; ++c) {
    const int it = tt * kNbChunks + c;
    const int s = it % kNbStages;
    const uint32_t ph = (it / kNbStages) & 1;
    mbar_wait(&full[s], ph, status, 710 + s);
    const uint32_t st = base + s * kNbStageBytes;
    const uint64_t q_hi = gmma_desc_sw128(st + g * 64 * 128), q_lo = gmma_desc_sw128(st + kNbATile + g * 64 * 128);
    const uint64_t r_hi = gmma_desc_sw128(st + 2 * kNbATile), r_lo = gmma_desc_sw128(st + 2 * kNbATile + kNbBTile);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kNbBK / 8; ++kk) {                   // K = 8 TF32 = 32 bytes per instruction
      wgmma_tf32_n192(d, q_hi + kk * 2, r_hi + kk * 2, (c == 0 && kk == 0) ? 0u : 1u);
      wgmma_tf32_n192(d, q_lo + kk * 2, r_hi + kk * 2, 1u);
      wgmma_tf32_n192(d, q_hi + kk * 2, r_lo + kk * 2, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);                      // the stage may be refilled
  }
  wgmma_fence_regs(d);
}

__global__ void __launch_bounds__(kNbThreads, 1)
nb_search_kernel(const __grid_constant__ CUtensorMap tm_q_hi, const __grid_constant__ CUtensorMap tm_q_lo,
                 const __grid_constant__ CUtensorMap tm_r_hi, const __grid_constant__ CUtensorMap tm_r_lo, const NbSearchParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int k = p.k;
  float* lsim = reinterpret_cast<float*>(smem + kNbStages * kNbStageBytes);     // [128 queries][k]
  int* lidx = reinterpret_cast<int*>(lsim + kNbBM * k);
  uint64_t* full = reinterpret_cast<uint64_t*>(lidx + kNbBM * k);                // 8-byte aligned: 128 k is even
  uint64_t* empty = full + kNbStages;                                             // one arrival per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // a 1-D grid, split fastest (the order of a (splits, query tiles) grid): gridDim.y would cap the query tiles at 65,535
  const int split = static_cast<int>(blockIdx.x % p.splits), m0 = static_cast<int>(blockIdx.x / p.splits) * kNbBM;
  const int t0 = split * p.tiles_per_split;
  const int nt = min(p.tiles_per_split, (p.n_ref + kNbBN - 1) / kNbBN - t0);    // >= 1 by construction of the grid

  if (warp == 0 && lane == 0) nb_ring_init(&tm_q_hi, &tm_q_lo, &tm_r_hi, &tm_r_lo, full, empty);
  for (int i = threadIdx.x; i < kNbBM * k; i += kNbThreads) { lsim[i] = -CUDART_INF_F; lidx[i] = -1; }
  __syncthreads();

  if (warp == 0 && lane == 0) {
    // ===================================================================== TMA producer
    nb_produce(&tm_q_hi, &tm_q_lo, &tm_r_hi, &tm_r_lo, smem, full, empty, m0, t0, nt, p.status);
  } else if (warp >= 4) {
    // ===================================================================== MMA + top-k: warpgroup g owns queries 64 g .. 64 g + 63
    const int g = (warp >> 2) - 1, wq = warp & 3;
    const uint32_t base = smem_u32(smem);
    int rowl[2], self_col[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      rowl[h] = g * 64 + wq * 16 + (lane >> 2) + 8 * h;
      const long long c = p.self_off == LLONG_MIN ? -1 : static_cast<long long>(m0 + rowl[h]) + p.self_off;
      self_col[h] = (c >= 0 && c < p.n_ref) ? static_cast<int>(c) : -1;
    }
    float ws[2] = {-CUDART_INF_F, -CUDART_INF_F};
    int wi[2] = {-1, -1}, wp[2] = {k - 1, k - 1};
    float d[96];
    for (int tt = 0; tt < nt; ++tt) {
      nb_tile_mma(d, base, full, empty, g, tt, p.status);
      // ------------------------------------------------------------------- top-k: register i holds row 8 ((i >> 1) & 1) + ...,
      // column 8 (i >> 2) + 2 (lane % 4) + (i & 1) of the tile (wgmma.cuh)
      const int n0 = (t0 + tt) * kNbBN + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int j = 0; j < kNbBN / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float v = d[4 * j + 2 * h + e];
            if (__any_sync(0xffffffffu, v >= ws[h]))
              nb_offer(v, n0 + 8 * j + e, rowl[h], self_col[h], p.n_ref, k, ws[h], wi[h], wp[h], lsim, lidx);
          }
        }
      }
    }
    // ===================================================================== each row's list, sorted, to the workspace
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = m0 + rowl[h];
      if (q >= p.n_query) continue;
      const float* rs = lsim + rowl[h] * k;
      const int* ri = lidx + rowl[h] * k;
      const size_t o = (static_cast<size_t>(split) * p.n_query + q) * k;
      for (int a = lane & 3; a < k; a += 4) {
        const float s = rs[a]; const int i = ri[a];
        int rank = 0;
        for (int b = 0; b < k; ++b) rank += nb_beats(rs[b], ri[b], s, i) || (b < a && rs[b] == s && ri[b] == i);   // equal: pads
        p.part_sim[o + rank] = s;
        p.part_idx[o + rank] = i;
      }
    }
  }
}

// Merge two sorted lists of k entries held by a warp (slot x in register x >> 5 of lane x & 31; pads (-inf, -1) beyond a
// list's end) into `a`.  An entry's place in the merged list is its slot plus the number of entries of the other list that
// rank before it (on equal keys, a's entries first): keys are distinct except the pads, which all carry the same value.
__device__ __forceinline__ void nb_merge_warp(float (&as)[2], long long (&ai)[2], const float (&bs)[2], const long long (&bi)[2],
                                              int k, float* ms, long long* mi) {
  const int lane = threadIdx.x & 31;
  int pa[2] = {lane, lane + 32}, pb[2] = {lane, lane + 32};
  for (int y = 0; y < k; ++y) {
    const int src = y & 31;
    const float ys = __shfl_sync(0xffffffffu, y < 32 ? bs[0] : bs[1], src);
    const long long yi = __shfl_sync(0xffffffffu, y < 32 ? bi[0] : bi[1], src);
    const float xs = __shfl_sync(0xffffffffu, y < 32 ? as[0] : as[1], src);
    const long long xi = __shfl_sync(0xffffffffu, y < 32 ? ai[0] : ai[1], src);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      pa[r] += nb_beats(ys, yi, as[r], ai[r]);         // b's entry y before a's entry
      pb[r] += !nb_beats(bs[r], bi[r], xs, xi);        // a's entry y before (or equal to) b's entry
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (lane + 32 * r < k && pa[r] < k) { ms[pa[r]] = as[r]; mi[pa[r]] = ai[r]; }
    if (lane + 32 * r < k && pb[r] < k) { ms[pb[r]] = bs[r]; mi[pb[r]] = bi[r]; }
  }
  __syncwarp();
#pragma unroll
  for (int r = 0; r < 2; ++r)
    if (lane + 32 * r < k) { as[r] = ms[lane + 32 * r]; ai[r] = mi[lane + 32 * r]; }
  __syncwarp();
}

// one warp per query: the splits' lists merged in split order; rows -> global indices (ref_index0 + row)
__global__ void __launch_bounds__(256) nb_finalize_kernel(const float* __restrict__ part_sim, const int32_t* __restrict__ part_idx,
                                                          int splits, int n_query, int k, long long ref_index0, float* out_sim,
                                                          long long* out_idx) {
  __shared__ float ms[8][kNbMaxK];
  __shared__ long long mi[8][kNbMaxK];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * 8 + w;
  if (q >= n_query) return;
  float as[2] = {-CUDART_INF_F, -CUDART_INF_F};
  long long ai[2] = {-1, -1};
  for (int s = 0; s < splits; ++s) {
    float bs[2] = {-CUDART_INF_F, -CUDART_INF_F};
    long long bi[2] = {-1, -1};
    const size_t o = (static_cast<size_t>(s) * n_query + q) * k;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int x = lane + 32 * r;
      if (x < k) {
        const int i = part_idx[o + x];
        bs[r] = part_sim[o + x];
        bi[r] = i < 0 ? -1 : ref_index0 + i;
        if (i < 0) bs[r] = -CUDART_INF_F;
      }
    }
    nb_merge_warp(as, ai, bs, bi, k, ms[w], mi[w]);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int x = lane + 32 * r;
    if (x < k) { out_sim[static_cast<size_t>(q) * k + x] = as[r]; out_idx[static_cast<size_t>(q) * k + x] = ai[r]; }
  }
}

// one warp per query: (sim, idx) <- merge of (sim, idx) and (sim_b, idx_b)
__global__ void __launch_bounds__(256) nb_merge_kernel(float* sim, long long* idx, const float* __restrict__ sim_b,
                                                       const long long* __restrict__ idx_b, int n_query, int k) {
  __shared__ float ms[8][kNbMaxK];
  __shared__ long long mi[8][kNbMaxK];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * 8 + w;
  if (q >= n_query) return;
  float as[2] = {-CUDART_INF_F, -CUDART_INF_F}, bs[2] = {-CUDART_INF_F, -CUDART_INF_F};
  long long ai[2] = {-1, -1}, bi[2] = {-1, -1};
  const size_t o = static_cast<size_t>(q) * k;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int x = lane + 32 * r;
    if (x < k) { as[r] = sim[o + x]; ai[r] = idx[o + x]; bs[r] = sim_b[o + x]; bi[r] = idx_b[o + x]; }
  }
  nb_merge_warp(as, ai, bs, bi, k, ms[w], mi[w]);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int x = lane + 32 * r;
    if (x < k) { sim[o + x] = as[r]; idx[o + x] = ai[r]; }
  }
}

}  // namespace gnm
