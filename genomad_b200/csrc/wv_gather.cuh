// K3 + K4 fused: the IGLOO value projection q = maxpool8(y @ w_v) on the tensor cores (wgmma) AND the IGLOO patch gather
// mpi[p] = sum_k y[P[p,k],:] . Wf[p,k,:], in ONE pass over the activations (replaces conv_t_kernel<true> + patch_stream_kernel,
// which each stream the same hi16/lo16 planes from HBM).
//
// Reference semantics (genomad/neural_network/igloo.py:190-214):
//   mpi   = gather_nd(transpose(y), patches) * w_mult, reshaped, @ w_summer + w_bias          (lines 192-206)
//   y_proj = y @ w_v, MaxPool1D(8)                                                              (lines 208-210)
//
// Work decomposition: POSITION BANDS.  A unit is one band of 24 consecutive positions of 8 consecutive windows
// (192 activation rows; 250 bands x ceil(n/8) window groups).  Units are numbered band-major and every CTA owns a contiguous
// range of them, so a CTA stays on one band (at most three) for the whole launch while the grid as a whole sweeps the windows
// front to back.  That is what makes the gather cheap here: the ~34 (patch, slot) entries whose position falls into the CTA's
// band use the same 17 KB of folded weights for every unit (L1 / L2 resident), instead of every window re-reading all 4.3 MB.
//
// Slab.  The four regions of a unit (hi16 / lo16 plane x channel half) are ONE 3-D TMA box each, from a tensor map that lists
// the window axis BEFORE the position axis (api.cu make_band_map): the box {128 B, 8 windows, 24 positions} lands as
// [position][window][128 B], i.e. the 8 windows of one position are one 1024-byte swizzle atom.  For the tensor core the
// region is still a plain K-major SWIZZLE_128B operand of 192 rows (column n = 8 * position + window); for the gather it means
// "one position x 8 windows" is one conflict-free ldmatrix.  Six region buffers: the TMA producer fills the first half of unit
// u+1 while the MMAs and the gather work on unit u.
//
//   * value projection: 3 fp16 passes Ahi*Whi + Alo*Whi + Ahi*Wlo, operands swapped so that D^T[cout][row].  The w_v weights
//     (the A operand, 64 KB: hi / lo x two K-halves) are loaded into shared memory once per CTA.  Two MMA warpgroups own 64
//     output channels each and take the unit one pool group (64 columns = 8 positions x 8 windows) at a time, M64 N64 K16:
//     a thread's 32 accumulator registers hold 2 channels x 2 windows x the group's 8 positions, so the max-pool is a max over
//     8 of its own registers and q is written straight from them.
//   * patch gather: warp-level mma.sync.m16n8k16 on the slab rows.  Entries are grouped by position (<= 4 per group;
//     8,400 entries hit ~4,500 positions).  For one group and one channel half, A[16 x 64] = the position's 8 windows' hi16 rows
//     (rows 0-7) and lo16 rows (rows 8-15), read by 4 ldmatrix.x4; B[64 x 8] = the fp16 hi / lo halves of the group's folded
//     weights (host-packed in fragment order, scaled by a power of two so the lo halves stay normal; L1 / L2 resident); the sum of
//     the four D entries of (window, entry) is (hi + lo) . (w_hi + w_lo) with fp32 accumulation -- the fp32-equivalent dot product.
//     15 gather warps take <= 2 groups each; pass 0 (channels 0-63) waits in registers, pass 1 adds channels 64-127 and writes
//     part_t[slot][window] (8 lanes = 32 contiguous bytes).  A region goes back to the producer when the 8 MMA warps and all 15
//     gather warps have arrived (count 23).  patch_finish_t_kernel adds a patch's four slots in fixed order k = 0..3 plus the bias.
//
// Warp roles (768 threads, 1 CTA per SM):  warps 0..7: two MMA + epilogue warpgroups | warps 8..22: patch gather |
// warp 23 lane 0: barrier init, the weight load and the activation producer (TMA).
#pragma once
#include <cuda.h>
#include <type_traits>
#include "common.cuh"
#include "conv_t.cuh"
#include "igloo.cuh"

namespace gnm {

constexpr int kBandRows   = 24;                                   // positions per band (multiple of the pool size 8)
constexpr int kBandWins   = 8;                                    // windows per unit
constexpr int kWgN        = kBandRows * kBandWins;                // activation rows per unit (192)
constexpr int kNumBands   = (kTok + kBandRows - 1) / kBandRows;   // 250 (the last band holds 21 valid rows)
constexpr int kWgRegion   = kWgN * 128;                           // bytes per slab region (192 rows x 128 B)               =  24576
constexpr int kWgBufs     = 6;                                    // region buffers: region k of unit `it` lives in buffer (4 it + k) % 6,
                                                                  // so the TMA fills the next unit's first K-half while this one is in use
constexpr int kWgSlab     = kWgBufs * kWgRegion;                  //                                                        = 147456
constexpr int kWgWBytes   = kWvStages * kBStage;                  // w_v^T hi / lo x two K-halves, the A operand            =  65536
constexpr int kWgMmaWarps = 8;                                    // two MMA + epilogue warpgroups
constexpr int kWgWarps    = 15;                                   // patch-gather warps (24 warps in all: 80 registers per thread)
constexpr int kWgThreads  = (kWgMmaWarps + kWgWarps + 1) * 32;    // 768
constexpr int kWgGroupCap = 2;                                    // position groups per warp on the fast path (30 per band; a band has <= 24
                                                                  // positions, so only positions with more than 4 entries can exceed it)
constexpr int kWgGroupMax = 4;                                    // entries per position group: the 8 columns of mma.m16n8k16 = 4 entries x (hi, lo)
constexpr int kWgSmem     = kWgSlab + kWgWBytes + 2048;           //                                                        = 215040
static_assert(kWgSmem <= 232448, "wv_gather_kernel exceeds the 227 KB of shared memory a CTA may use");
static_assert(kWgN == 3 * 64 && kBandRows == 3 * kPool && kBandWins == 8, "unit shape: three pool groups of 8 positions x 8 windows");
static_assert(kWgRegion % 1024 == 0, "regions must keep the 1024-byte alignment of the 128-byte swizzle");

struct WvGatherParams {
  float* q_out;                // [n][749][128]
  float out_scale;             // 1/32 (activation scale)
  const int2* grp;             // [groups of all bands] {first entry slot, row inside the band | entries << 8}: the entries (<= 4) on one position
  const int32_t* band_gstart;  // [kNumBands + 1] first position group of every band
  const uint4* wfrag;          // [kGsSlots][2 K-halves][4 k-steps][4 tig] folded weights * 2^k as mma.m16n8k16 B fragments {hi b0, hi b1, lo b0, lo b1}: a lane reads the (b0, b1) pair of its column
  float gather_unscale;        // 1 / (power of two that moved the folded weights into fp16's normal range)
  float* part_t;               // [kGsSlots][n_pad] per-entry dot products (slot-major: a unit's 8 windows are contiguous)
  int n_windows, n_pad;        // n_pad = n rounded up to a multiple of 8
  int groups;                  // window groups per band = n_pad / 8
  int n_units;                 // kNumBands * groups
  const int32_t* cta_split;    // [gridDim.x + 1] unit range of every CTA (api.cu wv_split: near-equal unit counts)
  int experiment;              // timing experiments only (results become wrong): 32 = no gather work, 64 = no part_t stores, 128 = no q stores, 256 = gather reads its rows and weights but does no arithmetic, 1024 = no folded-weight loads, 2048 = no ldmatrix
  long long* dbg;              // optional [gridDim.x][8] cycle counters (nullptr = off), see tools/ab_stages.py --wvg-cycles
  DeviceStatus* status;
};

__device__ __forceinline__ uint2 ldg_frag(const uint2* p) {          // folded-weight fragments: keep them in L1 across units
  uint2 v;
  asm volatile("ld.global.nc.L1::evict_last.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}
// four 8x8 fp16 matrices; lanes 8i..8i+7 give the row addresses of matrix i, register i of lane l = matrix i [l / 4][2 (l % 4) .. +1]
__device__ __forceinline__ void ldsm_x4(uint32_t saddr, uint32_t (&a)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"(saddr));
}
// D[16x8] += A[16x16] * B[16x8], fp16 operands, fp32 accumulation (warp-level tensor-core instruction)
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(kWgThreads, 1)
wv_gather_kernel(const __grid_constant__ CUtensorMap tm_band, const __grid_constant__ CUtensorMap tm_w, const WvGatherParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_a = smem;                                   // ring of kWgBufs region buffers, each [24 positions][8 windows] x 128 B
  uint8_t* s_w = smem + kWgSlab;                         // w_v stages (K-half, hi / lo), [128 cout][128 B] each
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_w + kWgWBytes);
  uint64_t* a_full = bars;            // [kWgBufs]  per buffer
  uint64_t* a_empty = bars + 8;       // [kWgBufs]
  uint64_t* w_full = bars + 16;       // [1]
  // Region k of a unit (need order: 0 hi16.k0, 1 lo16.k0, 2 hi16.k1, 3 lo16.k1) is load number g = 4 * it + k of this CTA and
  // lives in buffer g % kWgBufs; every role walks the buffers in the same order, so each keeps the first buffer of the
  // current unit (b0, advanced by 4 mod kWgBufs per unit) and one phase bit per buffer that it flips after each use.

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kProducerWarp = kWgMmaWarps + kWgWarps;
  // contiguous range of band-major unit numbers; the split points weigh a unit by its band's entry count (host side)
  const int u_begin = p.cta_split[blockIdx.x], u_end = p.cta_split[blockIdx.x + 1];

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&tm_band);
    tma_prefetch_desc(&tm_w);
    for (int i = 0; i < kWgBufs; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], kWgMmaWarps + kWgWarps); }
    mbar_init(w_full, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kProducerWarp && lane == 0) {
    // ===================================================================== weights (once), then the activation producer
    mbar_arrive_expect_tx(w_full, kWgWBytes);
    for (int q = 0; q < kWvStages; ++q) tma_load_2d_hint(s_w + q * kBStage, &tm_w, w_full, 0, q * 128, l2_policy_evict_last());
    const uint64_t pol = l2_policy_evict_first();
    uint32_t phases = 0;                                   // bit b: parity of buffer b's next "empty" wait is phase ^ 1
    int b0 = 0;
    for (int unit = u_begin; unit < u_end; ++unit) {
      const int band = unit / p.groups;
      const int w0 = (unit - band * p.groups) * kBandWins;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        int b = b0 + k; if (b >= kWgBufs) b -= kWgBufs;
        mbar_wait(&a_empty[b], ((phases >> b) & 1) ^ 1, p.status, 500 + b);
        phases ^= 1u << b;
        mbar_arrive_expect_tx(&a_full[b], kWgRegion);
        // k: 0 hi16 channels 0-63, 1 lo16 channels 0-63, 2 hi16 channels 64-127, 3 lo16 channels 64-127 (byte offset in the row)
        const int src = (k & 1 ? kOffLo16 : kOffHi16) + (k >> 1) * 128;
        tma_load_3d_hint(s_a + b * kWgRegion, &tm_band, &a_full[b], src, w0, band * kBandRows, pol);     // box = {128 B, 8 windows, 24 positions}
      }
      b0 += 4; if (b0 >= kWgBufs) b0 -= kWgBufs;
    }
  } else if (warp < kWgMmaWarps) {
    // ===================================================================== MMA + epilogue (warpgroup g: channels 64 g .. 64 g + 63)
    const int g = warp >> 2, wq = warp & 3;
    const uint32_t a_base = smem_u32(s_a);
    const uint32_t w_base = smem_u32(s_w) + g * 64 * 128;
    const int ch0 = g * 64 + wq * 16 + (lane >> 2);        // accumulator rows of this thread: channels ch0 and ch0 + 8
    const int win0 = 2 * (lane & 3);                       // accumulator columns: windows win0, win0 + 1 of every position
    const float oscale = p.out_scale;
    mbar_wait(w_full, 0, p.status, 510);
    uint32_t phases = 0;
    int b0 = 0;
    float d[32];
    for (int unit = u_begin; unit < u_end; ++unit) {
      const int band = unit / p.groups;
      const int w0 = (unit - band * p.groups) * kBandWins;
      int bufs[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        int b = b0 + k; if (b >= kWgBufs) b -= kWgBufs;
        bufs[k] = b;
        mbar_wait(&a_full[b], (phases >> b) & 1, p.status, 530 + b);
        phases ^= 1u << b;
      }
#pragma unroll 1
      for (int pg = 0; pg < kBandRows / kPool; ++pg) {          // pool group pg = rows 64 pg .. 64 pg + 63 of every region
        wgmma_fence();
#pragma unroll 1
        for (int kh = 0; kh < 2; ++kh) {
          const uint64_t yh = gmma_desc_sw128(a_base + bufs[2 * kh] * kWgRegion + pg * 64 * 128);       // B: hi16 rows
          const uint64_t yl = gmma_desc_sw128(a_base + bufs[2 * kh + 1] * kWgRegion + pg * 64 * 128);   // B: lo16 rows
          const uint64_t whi = gmma_desc_sw128(w_base + (2 * kh) * kBStage);                            // A: w_v^T hi
          const uint64_t wlo = gmma_desc_sw128(w_base + (2 * kh + 1) * kBStage);                        // A: w_v^T lo
          // the order of conv_t_kernel<true> and layer1_wv_kernel, so that all three produce bit-identical q
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            wgmma_f16_n64(d, whi + kk * 2, yh + kk * 2, (kh == 0 && kk == 0) ? 0u : 1u);
            wgmma_f16_n64(d, whi + kk * 2, yl + kk * 2, 1u);
          }
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_f16_n64(d, wlo + kk * 2, yh + kk * 2, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(d);
        // register 4 i + 2 h + e = channel ch0 + 8 h, position i of the pool group, window win0 + e
        const int gg = band * (kBandRows / kPool) + pg;
        if (gg < kPooled && !(p.experiment & 128)) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float m = d[2 * h + e];
#pragma unroll
              for (int i = 1; i < kPool; ++i) m = fmaxf(m, d[4 * i + 2 * h + e]);
              const int w = w0 + win0 + e;
              if (w < p.n_windows) p.q_out[(static_cast<size_t>(w) * kPooled + gg) * kC + ch0 + 8 * h] = m * oscale;
            }
        }
      }
      __syncwarp();
      if (lane == 0)
#pragma unroll
        for (int k = 0; k < 4; ++k) mbar_arrive(&a_empty[bufs[k]]);
      b0 += 4; if (b0 >= kWgBufs) b0 -= kWgBufs;
    }
  } else if (warp >= kWgMmaWarps && warp < kWgMmaWarps + kWgWarps) {
    // ===================================================================== patch gather
    const int gw = warp - kWgMmaWarps;                         // 0..14
    const float gscale = p.gather_unscale;
    // Gather lane roles.  ldmatrix: lanes 8i..8i+7 address matrix i = (plane i & 1: 0 hi16 / 1 lo16, 16-byte chunk i >> 1 of the
    // k-step), row lane & 7 = window.  The A fragment then holds rows 0..7 = the 8 windows' hi16 halves and rows 8..15 = their
    // lo16 halves; mma: gid = lane >> 2 = window (A / D row) = entry (B column), tig = lane & 3.
    const int lm_plane = (lane >> 3) & 1, lm_chunk = lane >> 4, lm_win = lane & 7;
    const int gid = lane >> 2, tig = lane & 3;
    const uint32_t slab = smem_u32(s_a);
    int it = 0;
    uint32_t phases = 0;
    int b0 = 0;
    long long c_wait_full = 0, c_gather = 0, tq = 0;
    const long long t_begin = clock64();
    int cur_band = -1, g_first = 0, g_cnt = 0, n_mine = 0;
    int my_e0[kWgGroupCap] = {0, 0}, my_meta[kWgGroupCap] = {0, 0};     // this warp's position groups of the band, fast path
    bool fast = true;
    // One position group x one K-half: D[16 x 8] = A[16 x 64] * B[64 x 8] as 4 independent k-steps.  B's
    // columns are (entry 0 hi, entry 0 lo, entry 1 hi, ...): the fp16 hi / lo halves of up to 4 entries' folded weights.  Returns
    // entry tig of window gid: (hi16 row + lo16 row) x (hi-weight column + lo-weight column).
    auto gather_group = [&](int e0, int meta, int kh, uint32_t hi_base, uint32_t lo_base) -> float {
      const int row = meta & 31, ne = meta >> 8;
      const uint2* wf = reinterpret_cast<const uint2*>(p.wfrag) + ((static_cast<size_t>(e0 + (gid >> 1)) * 2 + kh) * 16 + tig) * 2 + (gid & 1);
      uint2 b[4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) b[ks] = ((gid >> 1) < ne && !(p.experiment & 1024)) ? ldg_frag(wf + ks * 8) : make_uint2(0u, 0u);
      const uint32_t rb = (lm_plane ? lo_base : hi_base) + row * (kBandWins * 128) + lm_win * 128;
      uint32_t a[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        if (p.experiment & 2048) { a[ks][0] = a[ks][1] = a[ks][2] = a[ks][3] = rb; continue; }
        ldsm_x4(rb + (((ks * 2 + lm_chunk) ^ lm_win) << 4), a[ks]);     // 128-byte swizzle: chunk j -> j ^ (row & 7)
      }
      // four independent accumulators: the warp-level mma shares the tensor pipe with the wgmma stream, so no mma of a group
      // depends on another one
      float d[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) d[ks][0] = d[ks][1] = d[ks][2] = d[ks][3] = 0.f;
      if (p.experiment & 256) {                              // timing experiment: rows and weights are read, no arithmetic
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) asm volatile("" :: "r"(a[ks][0] | a[ks][1] | a[ks][2] | a[ks][3] | b[ks].x | b[ks].y));
      } else {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) mma_16816(d[ks], a[ks], b[ks].x, b[ks].y);
      }
      float v = 0.f;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) v += (d[ks][0] + d[ks][2]) + (d[ks][1] + d[ks][3]);      // fixed order
      return v * gscale;
    };
    for (int unit = u_begin; unit < u_end; ++unit, ++it) {
      const int band = unit / p.groups;
      const int w0 = (unit - band * p.groups) * kBandWins;
      if (band != cur_band) {                                  // this warp's position groups of the band: gw, gw + 15, ...
        cur_band = band;
        g_first = p.band_gstart[band];
        g_cnt = (p.experiment & 32) ? 0 : p.band_gstart[band + 1] - g_first;
        fast = g_cnt <= kWgWarps * kWgGroupCap;
        n_mine = 0;
#pragma unroll
        for (int i = 0; i < kWgGroupCap; ++i) {
          const int gi = gw + i * kWgWarps;
          if (fast && gi < g_cnt) { const int2 m = p.grp[g_first + gi]; my_e0[i] = m.x; my_meta[i] = m.y; n_mine = i + 1; }
        }
      }
      // ---------------- gather: this warp's position groups x the unit's 8 windows, one K-half per pass (the MMAs' order, so a
      // K-half's two regions go back to the producer while the other K-half is still in use)
      float c0[kWgGroupCap];                                   // pass-0 halves of the fast path
#pragma unroll 1
      for (int kh = 0; kh < 2; ++kh) {
        int bh = b0 + 2 * kh; if (bh >= kWgBufs) bh -= kWgBufs;               // buffer of this K-half's hi16 region
        int bl = b0 + 2 * kh + 1; if (bl >= kWgBufs) bl -= kWgBufs;           // ... and of its lo16 region
        const uint32_t ph_h = (phases >> bh) & 1, ph_l = (phases >> bl) & 1;
        phases ^= (1u << bh) | (1u << bl);
        const uint32_t hi_base = slab + bh * kWgRegion, lo_base = slab + bl * kWgRegion;
        if (p.dbg) tq = clock64();
        mbar_wait(&a_full[bh], ph_h, p.status, 550 + bh);          // hi16 K-half kh
        mbar_wait(&a_full[bl], ph_l, p.status, 560 + bl);          // lo16 K-half kh
        if (p.dbg) { const long long t = clock64(); c_wait_full += t - tq; tq = t; }
        if (fast) {
#pragma unroll
          for (int i = 0; i < kWgGroupCap; ++i)
            if (i < n_mine) {
              const float v = gather_group(my_e0[i], my_meta[i], kh, hi_base, lo_base);
              if (kh == 0) c0[i] = v;
              else if (tig < (my_meta[i] >> 8) && !(p.experiment & 64))         // 8 lanes (gid = window) write 32 contiguous bytes
                p.part_t[static_cast<size_t>(my_e0[i] + tig) * p.n_pad + w0 + gid] = c0[i] + v;
            }
        } else {
          // generic path (a band with more than 30 position groups: only patch sets that put more than 4 entries on many
          // positions): pass-0 halves are parked in part_t itself (the same thread reads them back in pass 1)
#pragma unroll 1
          for (int gi = gw; gi < g_cnt; gi += kWgWarps) {
            const int2 m = p.grp[g_first + gi];
            const float v = gather_group(m.x, m.y, kh, hi_base, lo_base);
            if (tig < (m.y >> 8)) {
              float* gp = p.part_t + static_cast<size_t>(m.x + tig) * p.n_pad + w0 + gid;
              *gp = kh == 0 ? v : *gp + v;
            }
          }
        }
        __syncwarp();
        if (lane == 0) { mbar_arrive(&a_empty[bh]); mbar_arrive(&a_empty[bl]); }           // this warp is done with the K-half's regions
        if (p.dbg) c_gather += clock64() - tq;
      }
      b0 += 4; if (b0 >= kWgBufs) b0 -= kWgBufs;
    }
    if (p.dbg && warp == kWgMmaWarps && lane == 0) {
      long long* d = p.dbg + blockIdx.x * 8;
      d[0] = clock64() - t_begin; d[1] = c_wait_full; d[2] = c_gather; d[5] = it;
    }
  }
}

// mpi[w][p] = ((part_t[s0][w] + part_t[s1][w]) + part_t[s2][w]) + part_t[s3][w] + bias[p],  s_k = slot_of[4p + k];
// also the value's two TF32 halves for the tensor-core logits GEMM (logits_tc.cuh).  32 patches x 32 windows per CTA;
// reads are contiguous along the window axis, the transposed tile makes the writes contiguous along the patch axis.
__global__ void __launch_bounds__(256)
patch_finish_t_kernel(const float* __restrict__ part_t, const int32_t* __restrict__ slot_of, const float* __restrict__ w_bias,
                      float* __restrict__ mpi, float* __restrict__ mpi_hi, float* __restrict__ mpi_lo, int n_windows, int n_pad) {
  __shared__ float tile[32][33];
  const int p0 = blockIdx.x * 32, w0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 8 rows of 32 threads
  for (int pp = ty; pp < 32; pp += 8) {
    const int pch = p0 + pp, w = w0 + tx;
    float v = 0.f;
    if (pch < kPatches && w < n_windows) {
      const int4 s4 = *reinterpret_cast<const int4*>(slot_of + pch * 4);
      v = (((part_t[static_cast<size_t>(s4.x) * n_pad + w] + part_t[static_cast<size_t>(s4.y) * n_pad + w]) +
            part_t[static_cast<size_t>(s4.z) * n_pad + w]) + part_t[static_cast<size_t>(s4.w) * n_pad + w]) + w_bias[pch];
    }
    tile[pp][tx] = v;
  }
  __syncthreads();
  for (int ww = ty; ww < 32; ww += 8) {
    const int pch = p0 + tx, w = w0 + ww;
    if (pch < kPatches && w < n_windows) {
      const float v = tile[tx][ww];
      const size_t o = static_cast<size_t>(w) * kPatches + pch;
      mpi[o] = v;
      const float hi = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
      mpi_hi[o] = hi;
      mpi_lo[o] = __uint_as_float(__float_as_uint(v - hi) & 0xffffe000u);
    }
  }
}

}  // namespace gnm
