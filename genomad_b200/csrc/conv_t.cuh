// K2/K3: causal Conv1D(128->128, k=6) + LeakyReLU, and the IGLOO value projection (y @ w_v, MaxPool1D(8)),
// as ONE persistent wgmma kernel template (conv_t_kernel<false> / conv_t_kernel<true>).
//
// Reference semantics:
//   Conv1D x2 + LeakyReLU(0.1)      genomad/neural_network/igloo.py:64-72
//         y'[t,:] = lrelu(b + sum_{j=0..5, t-5+j>=0} y[t-5+j,:] @ W[j])      W: [6][128 in][128 out]
//   y_proj = y @ w_v, MaxPool1D(8)  genomad/neural_network/igloo.py:208-210
//         q[g,:] = max_{r<8} (y[8g+r,:] @ Wv)     g < 749 (positions 5992..5996 are dropped)
//
// Arithmetic: fp32-equivalent split.  Every operand x is carried as hi = fp16(x) plus a correction
// lo = x - hi, and A*B is evaluated on the tensor cores as Ahi*Bhi + Alo*Bhi + Ahi*Blo with fp32
// accumulation in ONE accumulator (the dropped Alo*Blo term is ~2^-22).  tools/precision_study.py
// shows why a single TF32/fp16 pass is not enough for the 1e-4 parity bar (1.4e-4 worst case for the convs, 7e-4 for w_v).
//   * w_v (feeds max-pool -> mean -> BatchNorm with a 31x gain): all three passes in fp16, ~7e-6.
//   * convs: the main pass Ahi*Bhi in fp16; the two correction passes only need ~8 bits, so they run in
//     e4m3 (K = 32 per instruction: twice the rate) on pre-scaled operands.  All passes are
//     scaled to a common 2^S so they add up in the same accumulator, and the epilogue multiplies by 2^-S:
//         main  : (32*Ahi)            x fp16(W * 2^d)            S = 5 + d          (wmax * 2^d in (0.39, 0.78] * 2^16)
//         corr1 : e4m3(Alo * 2^12)    x e4m3(Whi * 2^(S-12))
//         corr2 : e4m3(Ahi * 2^7)     x e4m3(Wlo * 2^(S-7))
//     CPU emulation of exactly this recipe: max |dp| 6.5e-6 over 256 worst-case-family windows.
//
// Data layout.  Activation rows are 768 bytes: hi16 | lo16 | e4m3 pairs (lo8[c], hi8[c]) (common.cuh), tensor [n][5997][768 B].
// One work unit = 256 consecutive positions of one window (24 units per window).  The unit's operands
// are four slab REGIONS of 272 rows x 128 bytes (conv: hi16 ch 0-63, hi16 ch 64-127, e4m3 pairs of ch 0-63, of ch 64-127;
// w_v: hi16 and lo16 halves); two TMA boxes of 136 rows bring rows t0-5 .. t0+266 of the window into
// each SWIZZLE_128B region ONCE; conv tap j is the same slab read j rows further down -- only the
// wgmma descriptor start address changes (row j is position t0-5+j; TMA zero-fills rows with t < 0 or
// t >= 5997, which is exactly Keras' causal padding).
//
// Operand roles ("transposed" formulation).  The model has only 128 output channels, so the wide N = 256 side of the
// instruction comes from swapping the roles:
//
//     D^T[cout (M)][position (N=256)] += W_tap^T[cout][cin] * Y[position + tap][cin]
//
//   A operand = one 16 KB weight stage, [128 cout][64 cin] fp16 or [128 cout][128 cin] e4m3, K-major
//               SWIZZLE_128B, host-packed in consumption order; consumer warpgroup g multiplies its rows 64 g .. 64 g + 63,
//               which TMA streams as one contiguous 8 KB HALF-stage through warpgroup g's own ring of 5 slots;
//   B operand = 256 consecutive rows of one slab region.
//
// Schedule.  Weight stages are consumed region-major (all 6 taps against one region, then the next; the two e4m3 regions
// before the two fp16 ones, see the MMA loop) so a region is free after both warpgroups' 6 stages and is reloaded for the
// NEXT unit while the other regions are in use; activations and weights have separate producer threads.
// Ping-pong: ONE weight producer fills the two rings in the order (unit u, g = 0, all stages), (u, g = 1, all stages),
// (u + 1, g = 0, ...), ...  It can run at most 5 half-stages ahead of the warpgroup it is filling, so warpgroup 1 starts
// unit u when warpgroup 0 is ~5 stages from the end of it, and warpgroup 0 starts u + 1 when warpgroup 1 is ~5 stages from
// the end of u: each warpgroup's epilogue runs while its partner issues MMAs, and the tensor cores stay busy (one warpgroup
// has one warp on each SM sub-partition, so its M64 N256 stream alone can keep all four tensor cores busy).  The rings are
// separate because a waiter on an mbarrier must never be two phases ahead of it: in one ring shared by both warpgroups,
// warpgroup 1's first half-stage would take the slot and phase parity of a fill two laps earlier and pass its wait at once.
//
// Warp roles (384 threads = 3 warpgroups, 1 CTA per SM, persistent over units):
//   warpgroup 0: one elected thread of warp 0 produces the weights (TMA), one of warp 1 the activations (TMA)
//   warpgroups 1, 2: wgmma (M64 N256, 128 fp32 accumulator registers per thread) and the epilogue of output channels
//       64 g .. 64 g + 63.  A thread holds channels c and c + 8 at 64 of the unit's positions (wgmma.cuh).
//       conv : 2^-S scale + bias + LeakyReLU, then the planes the consumer needs (conv2 -> hi16, lo8, hi8 for
//              conv3; conv3 -> hi16, lo16 for w_v / gather).  Per column group of 8 positions a warp transposes its
//              16 channels x 8 positions x 2 planes through a private 512-byte shared-memory tile (one stmatrix.trans),
//              then each lane writes one full 16-byte half of a 32-byte sector: 32 st.global.v4 per thread and unit
//              instead of 512 two-byte stores, which is what lets the epilogue fit under the partner's MMA phase;
//       w_v  : the max over 8 consecutive positions (two registers per lane, then a butterfly over the lane quad).
//   The warpgroup index is broadcast from lane 0 and every stage of the MMA loop is unrolled at compile time, so ptxas sees
//   no divergent path between the wgmma of consecutive stages and keeps them in flight (wgmma_wait<1>) instead of draining
//   each one.
// The epilogue tracks the largest |Y| it produced and raises DeviceStatus::act_overflow beyond the operand formats' range.
// Option conv_cluster launches the persistent grid as thread-block clusters (every CTA still issues its own loads).
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace gnm {

constexpr int kTileM       = 128;
constexpr int kUnitsPerWin = (kTok + 2 * kTileM - 1) / (2 * kTileM);   // 24
constexpr int kSlabRows    = 136;                                // rows per TMA box
constexpr int kARegion     = kSlabRows * 128;                    // bytes per box: rows x 128 B            = 17408
constexpr int kA2Region    = 2 * kARegion;                       // 272-row slab region                    = 34816
constexpr int kNumRegions  = 4;
constexpr int kA2Bytes     = kNumRegions * kA2Region;            //                                        = 139264
constexpr int kBStage      = 128 * 128;                          // one weight stage: 128 rows x 128 B     = 16384
constexpr int kBHalf       = kBStage / 2;                        // one warpgroup's 64 rows of a stage     = 8192
constexpr int kConvThreads = 384;                                // producer warpgroup + 2 MMA / epilogue warpgroups
constexpr int kConvStages  = 24;                                 // conv: (region, tap)
constexpr int kWvStages    = 4;                                  // w_v : (K-half, weight hi/lo)
constexpr int kTWSlots     = 5;                                  // depth of each warpgroup's weight ring (8 KB half-stages)
constexpr int kEpiTile     = 512;                                // conv epilogue staging: 8 positions x 2 planes x 32 B per warp
constexpr int kEpiStage    = 8 * 2 * kEpiTile;                   // 8 consumer warps x 2 tiles (double-buffered)    = 8192
constexpr int kConvTSmem   = kA2Bytes + 2 * kTWSlots * kBHalf + kEpiStage + 2048;
static_assert(kConvTSmem <= 232448, "conv_t_kernel exceeds the 227 KB of shared memory a CTA may use");

struct ConvTcParams {
  const float* bias;        // [128] (conv) or nullptr (w_v)
  uint8_t* y_out;           // [n][5997][768 B] (conv) or nullptr
  float* q_out;             // [n][749][128] (w_v) or nullptr
  float out_scale;          // conv: 2^-S (undoes the common operand scaling); w_v: 2^-e / 32 (w_v operand scaling, activation scale)
  int out_fp8;              // conv: 1 = write hi16 + lo8 + hi8 (consumer is a conv), 0 = write hi16 + lo16
  int n_tiles;              // number of work units = n_windows * 24
  int experiment;           // timing experiments only (results become wrong): 2 = no epilogue global stores (the shared-memory transpose still runs)
  long long* dbg;           // optional [gridDim.x][8] cycle counters (nullptr = off)
  DeviceStatus* status;
};

// conv: consumption step q of a unit -> 16 KB stage of the host pack (packed region-major: hi16.k0, hi16.k1, pairs.k0, pairs.k1,
// six taps each), e4m3 regions first (see the MMA loop); w_v: the pack order
template <bool kWvMode> __device__ __forceinline__ int conv_pack_stage(int q) {
  return kWvMode ? q : ((q / 6 + 2) & 3) * 6 + q % 6;
}
// byte offset inside the 768-byte activation row of the data that fills slab region r
template <bool kWvMode> __device__ __forceinline__ constexpr int region_src(int r) {
  return kWvMode ? (r == 0 ? kOffHi16 : r == 1 ? kOffHi16 + 128 : r == 2 ? kOffLo16 : kOffLo16 + 128)
                 : (r == 0 ? kOffHi16 : r == 1 ? kOffHi16 + 128 : r == 2 ? kOffP8 : kOffP8 + 128);
}

// Epilogue modes of the kernel body.  kConvFwd / kConvWv are the forward's conv_t_kernel<false> / <true>.  The attribution
// pass (attr.cuh) adds two: kConvRoute is the w_v pass with an epilogue that also stores WHERE each pooled maximum sits, and
// kConvBwd is the conv pass run over time-reversed gradient rows against W[j]^T (no bias; lrelu' of the forward activation at the
// mirrored row; optional fp32 rows added first; fp32 output).  MMA loop, producers and rings are shared.
constexpr int kConvFwd = 0, kConvWv = 1, kConvRoute = 2, kConvBwd = 3;
struct ConvAttrExt {
  uint8_t* route_out;         // kConvRoute: [n][749][128] row (0..7) of each pooled maximum, the first one on ties
  const uint8_t* mask_rows;   // kConvBwd: forward activation rows [n][5997][768 B]; the sign of hi16 at row 5996 - r gives lrelu'
  const float* add_rows;      // kConvBwd: fp32 rows [n][5997][128] (natural order) added as s_w * add before the mask, or nullptr
  const float* s_w;           // kConvBwd: [n] per-window gradient scale (with add_rows)
  const float* s_in;          // kConvBwd: [n] per-window power of two the input rows carry on top of s_w, divided out, or nullptr
  float* f32_out;             // kConvBwd: fp32 rows [n][5997][128] at the mirrored (natural) row
  float* unit_max;            // kConvBwd: [n][24][8] max |output| per unit and consumer warp, or nullptr
};

template <int kMode>
__device__ __forceinline__ void conv_t_body(const CUtensorMap* tm_act_p, const CUtensorMap* tm_w_p, const ConvTcParams& p,
                                            const ConvAttrExt& x) {
  constexpr bool kWvMode = kMode == kConvWv || kMode == kConvRoute;
  constexpr int kStagesU = kWvMode ? kWvStages : kConvStages;     // stages per unit
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_a = smem;                                   // activation slab: 4 regions x 272 rows x 128 B
  uint8_t* s_w = smem + kA2Bytes;                        // weight rings of half-stages: [2 warpgroups][kTWSlots]
  uint8_t* s_epi = s_w + 2 * kTWSlots * kBHalf;          // conv epilogue staging tiles: [8 consumer warps][2][kEpiTile]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_epi + kEpiStage);
  uint64_t* a_full = bars;                      // [4]  per region
  uint64_t* a_empty = bars + 4;                 // [4]  one arrival per consumer warp of both warpgroups
  uint64_t* w_full = bars + 8;                  // [2][kTWSlots]
  uint64_t* w_empty = bars + 8 + 2 * kTWSlots;  // [2][kTWSlots]  one arrival per warp of the ring's warpgroup

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x) >> 5, 0);   // warp-uniform for the compiler
  const int wg = warp >> 2, wq = warp & 3, lane = threadIdx.x & 31;
  const int n_units = p.n_tiles;      // n_windows * 24

  if (threadIdx.x == 0) {
    tma_prefetch_desc(tm_act_p);
    tma_prefetch_desc(tm_w_p);
    for (int i = 0; i < kNumRegions; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 8); }
    for (int i = 0; i < 2 * kTWSlots; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (wq == 0 && elect_one()) {
      // =================================================================== weight producer: (unit, warpgroup, stage) order
      uint32_t wcount = 0;                                 // fills of each ring so far
      const uint64_t pol = l2_policy_evict_last();         // the 384 KB of weights are re-read by every CTA for every unit
      for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x, wcount += kStagesU)
        for (int g = 0; g < 2; ++g)
          for (int q = 0; q < kStagesU; ++q) {
            const int s = g * kTWSlots + (wcount + q) % kTWSlots;
            const uint32_t wphase = ((wcount + q) / kTWSlots) & 1;
            mbar_wait(&w_empty[s], wphase ^ 1, p.status, 110 + s);
            mbar_arrive_expect_tx(&w_full[s], kBHalf);
            tma_load_2d_hint(s_w + s * kBHalf, tm_w_p, &w_full[s], 0, conv_pack_stage<kWvMode>(q) * 128 + 64 * g, pol);
          }
    } else if (wq == 1 && elect_one()) {
      // =================================================================== activation producer
      int it = 0;
      const uint64_t pol = l2_policy_evict_first();        // activations stream through L2 once
      for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x, ++it) {
        const uint32_t ph = it & 1;
        const int w = unit / kUnitsPerWin;
        const int t0 = (unit - w * kUnitsPerWin) * (2 * kTileM);
#pragma unroll
        for (int k = 0; k < kNumRegions; ++k) {
          const int r = kWvMode ? (k == 0 ? 0 : k == 1 ? 2 : k == 2 ? 1 : 3) : (k + 2) & 3;   // order in which the MMAs need them
          mbar_wait(&a_empty[r], ph ^ 1, p.status, 100 + r);
          mbar_arrive_expect_tx(&a_full[r], kA2Region);
          uint8_t* dst = s_a + r * kA2Region;
          tma_load_3d_hint(dst, tm_act_p, &a_full[r], region_src<kWvMode>(r), t0 - 5, w, pol);
          tma_load_3d_hint(dst + kARegion, tm_act_p, &a_full[r], region_src<kWvMode>(r), t0 - 5 + kSlabRows, w, pol);
        }
      }
    }
  } else {
    // ===================================================================== MMA + epilogue (warpgroup g: channels 64 g .. 64 g + 63)
    const int g = wg - 1;
    const uint32_t a_base = smem_u32(s_a);
    const uint32_t w_base = smem_u32(s_w);
    const int ch0 = g * 64 + wq * 16 + (lane >> 2);        // accumulator rows of this thread: channels ch0 and ch0 + 8
    const float bias0 = (kWvMode || kMode == kConvBwd) ? 0.f : p.bias[ch0], bias1 = (kWvMode || kMode == kConvBwd) ? 0.f : p.bias[ch0 + 8];
    const float oscale = p.out_scale;
    float amax = 0.f;                                      // largest |Y| this thread produced (range check, common.cuh)
    int it = 0;
    long long w_a = 0, w_w = 0, t_mma = 0, t_epi = 0, tq;
    const long long t_begin = clock64();
    float d[128];
    for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x, ++it) {
      const uint32_t aph = it & 1;
      const int w = unit / kUnitsPerWin;
      const int t0 = (unit - w * kUnitsPerWin) * (2 * kTileM);
      const uint32_t wc0 = static_cast<uint32_t>(it) * kStagesU;           // fills of this warpgroup's ring before this unit
      const long long t_unit = clock64();
      // resources of the stage whose wgmma is still in flight: released once the next stage's wgmma is issued
      int prev_s = 0, prev_region = -1;
#pragma unroll
      for (int q = 0; q < kStagesU; ++q) {
        // conv: step q = (region ((q/6) + 2) % 4, tap q%6); regions 0,1 are fp16 K-halves, 2 / 3 = e4m3 pairs (lo8, hi8) of channels
        //       0-63 / 64-127 against weights interleaved the same way (Whi8, Wlo8).  The e4m3 correction passes run FIRST: the
        //       tensor core adds e4m3 products to the accumulator with less than fp32 precision, which would drop the ~2^-8 smaller
        //       corrections if the accumulator already held the main pass; the fp16 passes accumulate in full fp32.
        // w_v : stage q = (K-half q/2, weight hi/lo q%2); hi-weight stages multiply both the hi16 and the lo16 region
        // The loop is unrolled, so region, tap and instruction type are compile-time constants at every wgmma.
        const int reg = kWvMode ? (q >> 1) : ((q / 6 + 2) & 3);
        const int tap = kWvMode ? 5 : (q % 6);
        const bool first_use = kWvMode ? ((q & 1) == 0) : (tap == 0);
        if (first_use) {
          tq = clock64();
          mbar_wait(&a_full[reg], aph, p.status, 210 + reg);
          if (kWvMode) mbar_wait(&a_full[2 + reg], aph, p.status, 214 + reg);
          w_a += clock64() - tq;
        }
        const uint32_t c = wc0 + q;
        const int s = g * kTWSlots + c % kTWSlots;
        const uint32_t wphase = (c / kTWSlots) & 1;
        tq = clock64();
        mbar_wait(&w_full[s], wphase, p.status, 220 + s);
        w_w += clock64() - tq;
        const uint64_t wdesc = gmma_desc_sw128(w_base + s * kBHalf);                               // A: weights
        const uint64_t y0 = gmma_desc_sw128(a_base + reg * kA2Region + tap * 128);                 // B: activations
        wgmma_fence();
        int rel = -1;                                            // slab region this stage is the last user of
        if (kWvMode) {
          const uint64_t y1 = gmma_desc_sw128(a_base + (2 + reg) * kA2Region + tap * 128);        // lo16 region
          const bool w_lo = (q & 1) != 0;
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            wgmma_f16_n256(d, wdesc + kk * 2, y0 + kk * 2, (q == 0 && kk == 0) ? 0u : 1u);
            if (!w_lo) wgmma_f16_n256(d, wdesc + kk * 2, y1 + kk * 2, 1u);
          }
          rel = q == 0 ? 2 : q == 1 ? 0 : q == 2 ? 3 : 1;        // lo16.k0 is only used by stage 0, hi16.k0 by stages 0, 1, ...
        } else {
          if (reg >= 2) {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wgmma_e4m3_n256(d, wdesc + kk * 2, y0 + kk * 2, (q == 0 && kk == 0) ? 0u : 1u);
          } else {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wgmma_f16_n256(d, wdesc + kk * 2, y0 + kk * 2, 1u);
          }
          if (tap == 5) rel = reg;                               // this region of the slab is no longer needed
        }
        wgmma_commit();
        // the previous stage's wgmma has completed once at most one group (this stage's) is pending
        wgmma_wait<1>();
        if (q > 0) {
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&w_empty[prev_s]);
            if (prev_region >= 0) mbar_arrive(&a_empty[prev_region]);
          }
        }
        prev_s = s; prev_region = rel;
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&w_empty[prev_s]);
        if (prev_region >= 0) mbar_arrive(&a_empty[prev_region]);
      }
      wgmma_fence_regs(d);
      tq = clock64();
      t_mma += tq - t_unit;
      // ===================================================================== epilogue (overlaps the partner warpgroup's MMAs)
      if constexpr (kMode == kConvRoute) {
        // as below, with the row of the maximum carried along: a lane's two positions 2 (lane % 4) + e, then the lane quad;
        // a later row wins only if strictly larger, so ties go to the first row (the value is the forward's q bit for bit)
        const int r0 = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          float v[2];
          int ix[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float a = d[4 * j + 2 * h], b = d[4 * j + 2 * h + 1];
            v[h] = b > a ? b : a;
            ix[h] = b > a ? r0 + 1 : r0;
          }
#pragma unroll
          for (int off = 1; off <= 2; off <<= 1)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float pv = __shfl_xor_sync(0xffffffffu, v[h], off);
              const int pi = __shfl_xor_sync(0xffffffffu, ix[h], off);
              if (pv > v[h] || (pv == v[h] && pi < ix[h])) { v[h] = pv; ix[h] = pi; }
            }
          const int gg = (t0 >> 3) + j;
          if ((lane & 3) == 0 && gg < kPooled) {
            const size_t o = (static_cast<size_t>(w) * kPooled + gg) * kC;
            p.q_out[o + ch0] = v[0] * oscale;
            p.q_out[o + ch0 + 8] = v[1] * oscale;
            x.route_out[o + ch0] = static_cast<uint8_t>(ix[0]);
            x.route_out[o + ch0 + 8] = static_cast<uint8_t>(ix[1]);
          }
        }
      } else if (kWvMode) {
        // pool group j of the unit = accumulator columns 8 j .. 8 j + 7 = registers 4 j + 2 h + e of the lane quad
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          float m0 = fmaxf(d[4 * j], d[4 * j + 1]), m1 = fmaxf(d[4 * j + 2], d[4 * j + 3]);
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
          const int gg = (t0 >> 3) + j;
          if ((lane & 3) == 0 && gg < kPooled) {
            float* qrow = p.q_out + (static_cast<size_t>(w) * kPooled + gg) * kC;
            qrow[ch0] = m0 * oscale;
            qrow[ch0 + 8] = m1 * oscale;
          }
        }
      } else if constexpr (kMode == kConvBwd) {
        // backward pass into fp32 rows: accumulator row r is the gradient at position 5996 - r; plain 4-byte stores.  The input
        // scale s_in is a power of two, so dividing it out is exact; the unit maxima are order-free (deterministic)
        const float sw = x.add_rows ? x.s_w[w] : 0.f;
        const float inv = x.s_in ? 1.f / x.s_in[w] : 1.f;
        float umax = 0.f;
#pragma unroll
        for (int j = 0; j < 32; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int pos = t0 + 8 * j + 2 * (lane & 3) + e;
              if (pos < kTok) {
                const int ch = ch0 + 8 * h;
                const size_t row = static_cast<size_t>(w) * kTok + (kTok - 1 - pos);
                float v = d[4 * j + 2 * h + e] * oscale;
                if (x.s_in) v *= inv;
                if (x.add_rows) v = fmaf(sw, x.add_rows[row * kC + ch], v);
                const __half m = *reinterpret_cast<const __half*>(x.mask_rows + row * kRowBytes + kOffHi16 + 2 * ch);
                v = __hgt(m, __float2half(0.f)) ? v : v * kLeaky;
                x.f32_out[row * kC + ch] = v;
                umax = fmaxf(umax, fabsf(v));
              }
            }
        if (x.unit_max) {
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) umax = fmaxf(umax, __shfl_xor_sync(0xffffffffu, umax, off));
          if (lane == 0) x.unit_max[static_cast<size_t>(unit) * 8 + g * 4 + wq] = umax;
        }
      } else {
        // Column group j of the accumulator is this warp's 16 channels x 8 positions 8 j .. 8 j + 7.  Per output plane that is
        // 8 rows x 32 contiguous bytes, both planes 512 B: one 16-byte store per lane.  Both planes are b16 per (channel,
        // position) -- hi16 / lo16 halves, or the (lo8, hi8) e4m3 pair of a channel -- so the values of positions (pos, pos + 1)
        // are packed like a __half2, and one transposing stmatrix.x4 (matrix 2 k + h = plane k, channels ch0 + 8 h) turns the
        // fragment into position rows in the warp's staging tile: [position][plane][32 B], its 16-byte chunks XOR-swizzled by
        // position / 2 so that the stmatrix rows and the 16-byte reads are both free of bank conflicts.  The tile is
        // double-buffered, so the one __syncwarp between a tile's stmatrix and its reads also orders those reads before the
        // stmatrix that overwrites the tile two steps later.
        const bool store = !(p.experiment & 2);
        const uint32_t tile = smem_u32(s_epi) + (g * 4 + wq) * 2 * kEpiTile;
        const int sp = lane & 7, lp = lane >> 2;              // stmatrix row address of this lane / position it stores
        const uint32_t st_addr = tile + sp * 64 + (((lane >> 3) ^ (sp >> 1)) << 4);
        const uint32_t ld_addr = tile + lp * 64 + (((lane & 3) ^ (lp >> 1)) << 4);
        uint8_t* const dst = p.y_out + (static_cast<size_t>(w) * kTok + t0 + lp) * kRowBytes
                             + ((lane & 2) ? (p.out_fp8 ? kOffP8 : kOffLo16) : kOffHi16) + 2 * (g * 64 + wq * 16) + 16 * (lane & 1);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          uint32_t r[4];                                         // r[2 k + h]: plane k of channel ch0 + 8 h at 2 positions
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float bias = h ? bias1 : bias0;
            const float y0 = kActScale * lrelu(fmaf(d[4 * j + 2 * h], oscale, bias));
            const float y1 = kActScale * lrelu(fmaf(d[4 * j + 2 * h + 1], oscale, bias));
            amax = fmaxf(amax, fmaxf(fabsf(y0), fabsf(y1)));
            if (p.out_fp8) {
              const __half2 hh = __floats2half2_rn(y0, y1);
              const float2 f = __half22float2(hh);
              // e4m3 pair (lo8, hi8) of this channel at each of the two positions
              const uint32_t e0 = pack_e4m3x2((y0 - f.x) * kLo8Scale, f.x * kHi8Scale);
              const uint32_t e1 = pack_e4m3x2((y1 - f.y) * kLo8Scale, f.y * kHi8Scale);
              r[h] = pack_h2(__low2half(hh), __high2half(hh));
              r[2 + h] = e0 | (e1 << 16);
            } else {
              __half2 hh, l;
              split2_f16(y0, y1, hh, l);
              r[h] = pack_h2(__low2half(hh), __high2half(hh));
              r[2 + h] = pack_h2(__low2half(l), __high2half(l));
            }
          }
          const uint32_t buf = (j & 1) * kEpiTile;
          stmatrix_x4_trans(st_addr + buf, r[0], r[1], r[2], r[3]);
          __syncwarp();
          const uint4 v = ld_shared_v4(ld_addr + buf);
          if (store && t0 + 8 * j + lp < kTok) *reinterpret_cast<uint4*>(dst + static_cast<size_t>(8 * j) * kRowBytes) = v;
        }
      }
      t_epi += clock64() - tq;
    }
    if constexpr (!kWvMode && kMode != kConvBwd) flag_act_overflow(p.status, amax, p.out_fp8 ? kHi8Limit : kF16Limit, p.out_fp8 ? 2 : 3);
    if (p.dbg && wq == 0 && lane == 0) {     // include/gnm.h, "conv_dbg"
      long long* dd = p.dbg + blockIdx.x * 8;
      if (g == 0) { dd[0] = clock64() - t_begin; dd[1] = t_mma; dd[2] = w_a; dd[3] = w_w; dd[4] = it; dd[6] = t_epi; }
      else { dd[5] = t_mma; dd[7] = t_epi; }
    }
  }
}

// tm_w: the weight pack with a 64-row box, i.e. one warpgroup's half of a 16 KB stage per load
template <bool kWvMode>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_t_kernel(const __grid_constant__ CUtensorMap tm_act, const __grid_constant__ CUtensorMap tm_w,
              const ConvTcParams p) {
  conv_t_body<kWvMode ? kConvWv : kConvFwd>(&tm_act, &tm_w, p, ConvAttrExt{});
}

// the attribution pass's instantiations (attr.cuh): kMode = kConvRoute or kConvBwd
template <int kMode>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_t_attr_kernel(const __grid_constant__ CUtensorMap tm_act, const __grid_constant__ CUtensorMap tm_w,
                   const ConvTcParams p, const ConvAttrExt x) {
  conv_t_body<kMode>(&tm_act, &tm_w, p, x);
}

}  // namespace gnm
