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
//         main  : (32*Ahi)            x fp16(Whi * 2^d)          S = 5 + d          (d = 16 for |W| < 0.78)
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
//               SWIZZLE_128B (streamed by TMA through a 5-stage ring, host-packed in consumption order);
//               consumer warpgroup g multiplies its rows 64 g .. 64 g + 63;
//   B operand = 256 consecutive rows of one slab region.
//
// Schedule.  Weight stages are consumed region-major (all 6 taps against one region, then the next; the two e4m3 regions
// before the two fp16 ones, see the MMA loop) so a region is free after its 6 stages and is reloaded for the NEXT unit while
// the other regions are in use;
// activations and weights have separate producer threads.
//
// Warp roles (384 threads = 3 warpgroups, 1 CTA per SM, persistent over units):
//   warp 0 lane 0 : weight producer (TMA)          warp 1 lane 0 : activation producer (TMA)
//   warpgroups 1, 2: wgmma (M64 N256, 128 fp32 accumulator registers per thread) and the epilogue of output channels
//       64 g .. 64 g + 63.  A thread holds channels c and c + 8 at 64 of the unit's positions (wgmma.cuh).
//       conv : 2^-S scale + bias + LeakyReLU, then the planes the consumer needs (conv2 -> hi16, lo8, hi8 for
//              conv3; conv3 -> hi16, lo16 for w_v / gather) stored straight to global memory;
//       w_v  : the max over 8 consecutive positions (two registers per lane, then a butterfly over the lane quad).
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
constexpr int kConvThreads = 384;                                // producer warpgroup + 2 MMA / epilogue warpgroups
constexpr int kConvStages  = 24;                                 // conv: (region, tap)
constexpr int kWvStages    = 4;                                  // w_v : (K-half, weight hi/lo)
constexpr int kTWStages    = 5;                                  // weight ring depth (16 KB each)
constexpr int kConvTSmem   = kA2Bytes + kTWStages * kBStage + 2048;

struct ConvTcParams {
  const float* bias;        // [128] (conv) or nullptr (w_v)
  uint8_t* y_out;           // [n][5997][768 B] (conv) or nullptr
  float* q_out;             // [n][749][128] (w_v) or nullptr
  float out_scale;          // conv: 2^-S (undoes the common operand scaling); w_v: 1/32 (activation scale)
  int out_fp8;              // conv: 1 = write hi16 + lo8 + hi8 (consumer is a conv), 0 = write hi16 + lo16
  int n_tiles;              // number of work units = n_windows * 24
  int experiment;           // timing experiments only (results become wrong): 2 = no epilogue global stores
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

template <bool kWvMode>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_t_kernel(const __grid_constant__ CUtensorMap tm_act, const __grid_constant__ CUtensorMap tm_w,
              const ConvTcParams p) {
  constexpr int kStagesU = kWvMode ? kWvStages : kConvStages;     // stages per unit
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_a = smem;                                   // activation slab: 4 regions x 272 rows x 128 B
  uint8_t* s_w = smem + kA2Bytes;                        // weight ring
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_w + kTWStages * kBStage);
  uint64_t* a_full = bars;            // [4]  per region
  uint64_t* a_empty = bars + 4;       // [4]  one arrival per consumer warp
  uint64_t* w_full = bars + 8;        // [5]
  uint64_t* w_empty = bars + 13;      // [5]  one arrival per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_units = p.n_tiles;      // n_windows * 24

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_act);
    tma_prefetch_desc(&tm_w);
    for (int i = 0; i < kNumRegions; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 8); }
    for (int i = 0; i < kTWStages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 1 && lane == 0) {
    // ===================================================================== activation producer
    int it = 0;
    const uint64_t pol = l2_policy_evict_first();          // activations stream through L2 once
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
        tma_load_3d_hint(dst, &tm_act, &a_full[r], region_src<kWvMode>(r), t0 - 5, w, pol);
        tma_load_3d_hint(dst + kARegion, &tm_act, &a_full[r], region_src<kWvMode>(r), t0 - 5 + kSlabRows, w, pol);
      }
    }
  } else if (warp == 0 && lane == 0) {
    // ===================================================================== weight producer
    uint32_t wcount = 0;
    const uint64_t pol = l2_policy_evict_last();           // the 384 KB of weights are re-read by every CTA for every unit
    for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
      for (int q = 0; q < kStagesU; ++q, ++wcount) {
        const int s = wcount % kTWStages;
        const uint32_t wphase = (wcount / kTWStages) & 1;
        mbar_wait(&w_empty[s], wphase ^ 1, p.status, 110 + s);
        mbar_arrive_expect_tx(&w_full[s], kBStage);
        tma_load_2d_hint(s_w + s * kBStage, &tm_w, &w_full[s], 0, conv_pack_stage<kWvMode>(q) * 128, pol);
      }
    }
  } else if (warp >= 4) {
    // ===================================================================== MMA + epilogue (warpgroup g: channels 64 g .. 64 g + 63)
    const int g = (warp >> 2) - 1, wq = warp & 3;
    const uint32_t a_base = smem_u32(s_a);
    const uint32_t w_base = smem_u32(s_w) + g * 64 * 128;  // this warpgroup's 64 rows of every weight stage
    const int ch0 = g * 64 + wq * 16 + (lane >> 2);        // accumulator rows of this thread: channels ch0 and ch0 + 8
    const float bias0 = kWvMode ? 0.f : p.bias[ch0], bias1 = kWvMode ? 0.f : p.bias[ch0 + 8];
    const float oscale = p.out_scale;
    float amax = 0.f;                                      // largest |Y| this thread produced (range check, common.cuh)
    uint32_t wcount = 0;
    int it = 0;
    long long w_a = 0, w_w = 0, t_epi = 0, tq;
    const long long t_begin = clock64();
    float d[128];
    for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x, ++it) {
      const uint32_t aph = it & 1;
      const int w = unit / kUnitsPerWin;
      const int t0 = (unit - w * kUnitsPerWin) * (2 * kTileM);
      // resources of the stage whose wgmma is still in flight: released once the next stage's wgmma is issued
      int prev_s = -1, prev_region = -1;
      for (int q = 0; q < kStagesU; ++q, ++wcount) {
        // conv: step q = (region ((q/6) + 2) % 4, tap q%6); regions 0,1 are fp16 K-halves, 2 / 3 = e4m3 pairs (lo8, hi8) of channels
        //       0-63 / 64-127 against weights interleaved the same way (Whi8, Wlo8).  The e4m3 correction passes run FIRST: the
        //       tensor core adds e4m3 products to the accumulator with less than fp32 precision, which would drop the ~2^-8 smaller
        //       corrections if the accumulator already held the main pass; the fp16 passes accumulate in full fp32.
        // w_v : stage q = (K-half q/2, weight hi/lo q%2); hi-weight stages multiply both the hi16 and the lo16 region
        const int reg = kWvMode ? (q >> 1) : ((q / 6 + 2) & 3);
        const int tap = kWvMode ? 5 : (q % 6);
        const bool first_use = kWvMode ? ((q & 1) == 0) : (tap == 0);
        if (first_use) {
          tq = clock64();
          mbar_wait(&a_full[reg], aph, p.status, 210 + reg);
          if (kWvMode) mbar_wait(&a_full[2 + reg], aph, p.status, 214 + reg);
          w_a += clock64() - tq;
        }
        const int s = wcount % kTWStages;
        const uint32_t wphase = (wcount / kTWStages) & 1;
        tq = clock64();
        mbar_wait(&w_full[s], wphase, p.status, 220 + s);
        w_w += clock64() - tq;
        const uint64_t wdesc = gmma_desc_sw128(w_base + s * kBStage);                              // A: weights
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
          if (reg < 2) {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wgmma_f16_n256(d, wdesc + kk * 2, y0 + kk * 2, 1u);
          } else {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wgmma_e4m3_n256(d, wdesc + kk * 2, y0 + kk * 2, (q == 0 && kk == 0) ? 0u : 1u);
          }
          if (tap == 5) rel = reg;                               // this region of the slab is no longer needed
        }
        wgmma_commit();
        // the previous stage's wgmma has completed once at most one group (this stage's) is pending
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0 && prev_s >= 0) {
          mbar_arrive(&w_empty[prev_s]);
          if (prev_region >= 0) mbar_arrive(&a_empty[prev_region]);
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
      // ===================================================================== epilogue
      tq = clock64();
      if (kWvMode) {
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
      } else {
        const bool store = !(p.experiment & 2);
        uint8_t* const unit_rows = p.y_out + (static_cast<size_t>(w) * kTok + t0) * kRowBytes;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int pos = 8 * j + 2 * (lane & 3);                // positions pos, pos + 1 of the unit
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int ch = ch0 + 8 * h;
            const float bias = h ? bias1 : bias0;
            const float y0 = kActScale * lrelu(fmaf(d[4 * j + 2 * h], oscale, bias));
            const float y1 = kActScale * lrelu(fmaf(d[4 * j + 2 * h + 1], oscale, bias));
            amax = fmaxf(amax, fmaxf(fabsf(y0), fabsf(y1)));
            uint8_t* q0 = unit_rows + static_cast<size_t>(pos) * kRowBytes;
            uint8_t* q1 = q0 + kRowBytes;
            if (p.out_fp8) {
              const __half2 hh = __floats2half2_rn(y0, y1);
              const float2 f = __half22float2(hh);
              // e4m3 pair (lo8, hi8) of this channel at each of the two positions: one 2-byte store per position
              const uint16_t e0 = pack_e4m3x2((y0 - f.x) * kLo8Scale, f.x * kHi8Scale);
              const uint16_t e1 = pack_e4m3x2((y1 - f.y) * kLo8Scale, f.y * kHi8Scale);
              if (store && t0 + pos < kTok) {
                reinterpret_cast<__half*>(q0 + kOffHi16)[ch] = __low2half(hh);
                reinterpret_cast<uint16_t*>(q0 + kOffP8)[ch] = e0;
              }
              if (store && t0 + pos + 1 < kTok) {
                reinterpret_cast<__half*>(q1 + kOffHi16)[ch] = __high2half(hh);
                reinterpret_cast<uint16_t*>(q1 + kOffP8)[ch] = e1;
              }
            } else {
              __half2 hh, l;
              split2_f16(y0, y1, hh, l);
              if (store && t0 + pos < kTok) {
                reinterpret_cast<__half*>(q0 + kOffHi16)[ch] = __low2half(hh);
                reinterpret_cast<__half*>(q0 + kOffLo16)[ch] = __low2half(l);
              }
              if (store && t0 + pos + 1 < kTok) {
                reinterpret_cast<__half*>(q1 + kOffHi16)[ch] = __high2half(hh);
                reinterpret_cast<__half*>(q1 + kOffLo16)[ch] = __high2half(l);
              }
            }
          }
        }
      }
      t_epi += clock64() - tq;
    }
    if (!kWvMode) flag_act_overflow(p.status, amax, p.out_fp8 ? kHi8Limit : kF16Limit, p.out_fp8 ? 2 : 3);
    if (p.dbg && warp == 4 && lane == 0) {   // warpgroup 1's view
      long long* dd = p.dbg + blockIdx.x * 8;
      dd[0] = clock64() - t_begin; dd[2] = w_a; dd[3] = w_w; dd[4] = it; dd[6] = t_epi;
    }
  }
}

}  // namespace gnm
