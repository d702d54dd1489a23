// Layer 1 (tokens -> y1) fused with IGLOO#0's value projection q0 = maxpool8(y1 @ w_v#0).
//
// Reference semantics: OneHot + causal Conv1D(257->128, k=6) + LeakyReLU   genomad/neural_network/model.py:9-11, igloo.py:45-48
//                      y @ w_v, MaxPool1D(8)                                genomad/neural_network/igloo.py:207-210
//
// Why fuse: y1 is written once (4.7 GB per 1024 windows) and then read three times (patch gather, w_v, conv2).  The w_v
// read (3.1 GB) disappears if the projection consumes each row while it is still on the SM:
// the producer warps below write every finished row twice -- to global memory (all four planes, as embed_conv1_kernel
// does) and, as fp16 hi / lo halves, into a 128-byte-swizzled shared-memory slab in exactly the layout TMA would have
// produced -- and two warpgroups issue the same 3-pass wgmma conv_t_kernel<true> issues (D^T[cout][pos], weights as the
// A operand, the slab as the B operand).  The arithmetic of both halves is unchanged, so y1 and q0 are bit-identical to the
// unfused kernels' results.
//
// Persistent, 1 CTA per SM, 1024 threads:
//   warps 0-23  producers: tokens for the unit, then 4 rows each: two table rows from L2 -> y1 row ->
//               4 global plane stores + 2 swizzled shared stores; fence.proxy.async; arrive on a_full[buf]
//   warps 24-31 two MMA + epilogue warpgroups (output channels 64 g .. 64 g + 63): 2 x 24 wgmma M64 N48 K16 per unit, then
//               the max over 8 consecutive positions -> q0.  Warp 24 also initialises the barriers and loads w_v's four 16 KB
//               stages once (they stay resident).
// Unit = 96 positions (63 per window); the slab is double-buffered (2 x 4 regions x 12 KB), so producers fill unit u+1
// while the tensor core works on unit u.  Shared memory: 96 KB slab + 64 KB weights + barriers = 161 KB.
//
// Bit-identical to the two separate kernels (tests/test_gpu_parity.py::test_fused_layer1_wv_option); off by default
// (option "fuse_l1"): the producers are issue- and dependency-bound, so the fused kernel has not been faster than the pair.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "encode.cuh"

namespace gnm {

constexpr int kFuUnit = 96;                                      // positions per unit (two wgmma N = 48 halves)
constexpr int kFuUnitsPerWin = (kTok + kFuUnit - 1) / kFuUnit;   // 63
constexpr int kFuProducerWarps = 24;
constexpr int kFuRowsPerWarp = kFuUnit / kFuProducerWarps;      // 4, all loaded up front (8 table rows in flight per lane)
constexpr int kFuMmaWarps = 8;                                   // two MMA + epilogue warpgroups
constexpr int kFuThreads = 32 * (kFuProducerWarps + kFuMmaWarps);  // 1024
constexpr int kFuRegion = kFuUnit * 128;                         // 12 KB: 96 rows x 128 B (one K-half of one plane)
constexpr int kFuSlab = 4 * kFuRegion;                           // hi.k0 | hi.k1 | lo.k0 | lo.k1
constexpr int kFuWBytes = 4 * 16384;
constexpr int kFuSmem = 2 * kFuSlab + kFuWBytes + 256 + 1024;

struct FusedParams {
  const uint8_t* ascii;      // [n][6000] or nullptr
  const uint16_t* tokens;    // [n][5997] or nullptr
  const float* table;        // [6][257][128]
  const float* triple;       // [2][4096][128]
  const float* bias;         // [128]
  uint8_t* y_out;            // [n][5997][768 B]
  float* q_out;              // [n][749][128]
  int n_units;               // n_windows * 63
  DeviceStatus* status;
};

__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

template <bool kFromAscii>
__global__ void __launch_bounds__(kFuThreads, 1)
layer1_wv_kernel(const __grid_constant__ CUtensorMap tm_w, const FusedParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_slab = smem;                                  // [2][4][96 rows][128 B], 128B-swizzled
  uint8_t* s_w = smem + 2 * kFuSlab;                       // [4][128 rows][128 B]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_w + kFuWBytes);
  uint64_t* a_full = bars;            // [2]  count = producer warps
  uint64_t* a_empty = bars + 2;       // [2]  count = MMA warps
  uint64_t* w_full = bars + 4;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == kFuProducerWarps && lane == 0) {
    tma_prefetch_desc(&tm_w);
    for (int i = 0; i < 2; ++i) { mbar_init(&a_full[i], kFuProducerWarps); mbar_init(&a_empty[i], kFuMmaWarps); }
    mbar_init(w_full, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < kFuProducerWarps) {
    // ===================================================================== producers
    const float4 b4 = reinterpret_cast<const float4*>(p.bias)[lane];
    const float4* tab4 = reinterpret_cast<const float4*>(p.table);
    const float4* tri4 = reinterpret_cast<const float4*>(p.triple);
    auto add4 = [](float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); };
    auto row1 = [&](int j, int tk) -> float4 {
      return tk >= 0 ? __ldg(tab4 + (static_cast<size_t>(j) * kVocab + tk) * (kC / 4) + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    // A (taps 0..2) and B (taps 3..5) of the position whose six tokens start at tk[0]
    auto load_ab = [&](const int16_t* tk, float4& A, float4& B) {
      const int t0_ = tk[0], t1_ = tk[1], t2_ = tk[2], t3_ = tk[3], t4_ = tk[4], t5_ = tk[5];
      if (t0_ > 0 && t2_ > 0) A = __ldg(tri4 + static_cast<size_t>(((t0_ - 1) << 4) | ((t2_ - 1) & 15)) * (kC / 4) + lane);
      else A = add4(add4(row1(0, t0_), row1(1, t1_)), row1(2, t2_));
      if (t3_ > 0 && t5_ > 0) B = __ldg(tri4 + (static_cast<size_t>(kTriple) + (((t3_ - 1) << 4) | ((t5_ - 1) & 15))) * (kC / 4) + lane);
      else B = add4(add4(row1(3, t3_), row1(4, t4_)), row1(5, t5_));
    };
    const int kh = lane >> 4;                                      // which 64-channel K-half this lane's 4 channels are in
    const int chunk = (lane & 15) >> 1, sub = (lane & 1) * 8;      // 16-byte chunk inside the 128-byte half-row, 8-byte half
    // Every warp is autonomous (no CTA-wide barrier, no shared token buffer): lane 6r+j (r < 4, j < 6) computes the token of
    // position t-5+j of the warp's r-th row, rows read them by shuffle.  The warps of a CTA drift apart by up to the two slab
    // buffers, so one warp's table-load latency is another warp's compute time -- like the 8 CTAs per SM of the unfused kernel.
    const int my_r = lane / 6, my_j = lane - my_r * 6;             // lanes 24..31: idle in the token step
    auto unit_coords = [&](int unit, int& w, int& t0) { w = unit / kFuUnitsPerWin; t0 = (unit - w * kFuUnitsPerWin) * kFuUnit; };
    // bytes (or the token) for this lane's (row, tap) of `unit`; returns the token, -1 = causal pad / past the window end
    auto fetch_token = [&](int unit) -> int {
      if (lane >= 6 * kFuRowsPerWarp || unit >= p.n_units) return -1;
      int w, t0;
      unit_coords(unit, w, t0);
      const int pos = t0 + warp + my_r * kFuProducerWarps - 5 + my_j;
      if (pos < 0 || pos >= kTok) return -1;
      if (kFromAscii) {
        const uint8_t* src = p.ascii + static_cast<size_t>(w) * kWindow + pos;
        return kmer_token(base_code(__ldg(src)), base_code(__ldg(src + 1)), base_code(__ldg(src + 2)), base_code(__ldg(src + 3)));
      }
      return static_cast<int>(__ldg(p.tokens + static_cast<size_t>(w) * kTok + pos));
    };
    int it = 0;
    int tok_next = fetch_token(blockIdx.x);
    for (int unit = blockIdx.x; unit < p.n_units; unit += gridDim.x, ++it) {
      const int b = it & 1;
      const uint32_t ph = (it >> 1) & 1;
      int w, t0;
      unit_coords(unit, w, t0);
      const int tok_mine = tok_next;
      tok_next = fetch_token(unit + gridDim.x);                  // the next unit's bytes travel while this unit's rows are built
      int16_t tokv[kFuRowsPerWarp][6];
#pragma unroll
      for (int r = 0; r < kFuRowsPerWarp; ++r)
#pragma unroll
        for (int j = 0; j < 6; ++j) tokv[r][j] = static_cast<int16_t>(__shfl_sync(0xffffffffu, tok_mine, r * 6 + j));
      uint8_t* slab = s_slab + b * kFuSlab;
      // ---- 4 rows per warp (rows warp, warp+24, ...), all eight table rows requested before the first is used
      {
        float4 A[kFuRowsPerWarp], B[kFuRowsPerWarp];
#pragma unroll
        for (int r = 0; r < kFuRowsPerWarp; ++r) load_ab(tokv[r], A[r], B[r]);
        // ---- the slab buffer must have been consumed by the MMAs of unit it-2
        mbar_wait(&a_empty[b], ph ^ 1, p.status, 400 + b);
#pragma unroll
        for (int r = 0; r < kFuRowsPerWarp; ++r) {
          const int i = warp + r * kFuProducerWarps;
          const int t = t0 + i;
          float4 a = add4(A[r], B[r]);
          a.x = kActScale * lrelu(a.x + b4.x); a.y = kActScale * lrelu(a.y + b4.y);
          a.z = kActScale * lrelu(a.z + b4.z); a.w = kActScale * lrelu(a.w + b4.w);
          __half2 h01, h23, l01, l23;
          split2_f16(a.x, a.y, h01, l01);
          split2_f16(a.z, a.w, h23, l23);
          uint2 hv = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
          uint2 lv = make_uint2(*reinterpret_cast<const uint32_t*>(&l01), *reinterpret_cast<const uint32_t*>(&l23));
          if (t < kTok) {
            const float2 fa = __half22float2(h01), fb = __half22float2(h23);
            uint8_t* rowp = p.y_out + (static_cast<size_t>(w) * kTok + t) * kRowBytes;
            *reinterpret_cast<uint2*>(rowp + kOffHi16 + lane * 8) = hv;
            *reinterpret_cast<uint2*>(rowp + kOffLo16 + lane * 8) = lv;
            *reinterpret_cast<uint2*>(rowp + kOffP8 + lane * 8) = make_uint2(
                static_cast<uint32_t>(pack_e4m3x2((a.x - fa.x) * kLo8Scale, fa.x * kHi8Scale)) |
                    (static_cast<uint32_t>(pack_e4m3x2((a.y - fa.y) * kLo8Scale, fa.y * kHi8Scale)) << 16),
                static_cast<uint32_t>(pack_e4m3x2((a.z - fb.x) * kLo8Scale, fb.x * kHi8Scale)) |
                    (static_cast<uint32_t>(pack_e4m3x2((a.w - fb.y) * kLo8Scale, fb.y * kHi8Scale)) << 16));
          } else {
            hv = make_uint2(0u, 0u); lv = hv;          // columns past the window end: finite, ignored by the epilogue
          }
          // SWIZZLE_128B, K-major: row i of a region at i*128, its 16-byte chunk c stored at chunk c ^ (i & 7)
          const uint32_t off = static_cast<uint32_t>(i) * 128u + static_cast<uint32_t>((chunk ^ (i & 7)) * 16 + sub);
          *reinterpret_cast<uint2*>(slab + kh * kFuRegion + off) = hv;
          *reinterpret_cast<uint2*>(slab + (2 + kh) * kFuRegion + off) = lv;
        }
      }
      fence_proxy_async_smem();            // generic-proxy writes -> visible to the tensor core's async-proxy reads
      __syncwarp();
      if (lane == 0) mbar_arrive(&a_full[b]);
    }
  } else {
    // ===================================================================== MMA + epilogue (warpgroup g: channels 64 g .. 64 g + 63)
    const int g = (warp - kFuProducerWarps) >> 2, wq = warp & 3;
    if (warp == kFuProducerWarps && lane == 0) {           // the weights, once
      mbar_arrive_expect_tx(w_full, kFuWBytes);
      for (int q = 0; q < 4; ++q) tma_load_2d_hint(s_w + q * 16384, &tm_w, w_full, 0, q * 128, l2_policy_evict_last());
    }
    const uint32_t slab_base = smem_u32(s_slab), w_base = smem_u32(s_w) + g * 64 * 128;
    const int ch0 = g * 64 + wq * 16 + (lane >> 2);        // accumulator rows of this thread: channels ch0 and ch0 + 8
    const float oscale = 1.f / kActScale;
    mbar_wait(w_full, 0, p.status, 430);
    int it = 0;
    float d[24];
    for (int unit = blockIdx.x; unit < p.n_units; unit += gridDim.x, ++it) {
      const int b = it & 1;                                    // slab buffer
      const uint32_t ph = (it >> 1) & 1;
      const int w = unit / kFuUnitsPerWin;
      const int t0 = (unit - w * kFuUnitsPerWin) * kFuUnit;
      mbar_wait(&a_full[b], ph, p.status, 420 + b);
#pragma unroll 1
      for (int nh = 0; nh < 2; ++nh) {                          // positions 48 nh .. 48 nh + 47 of the unit (24 registers each)
        const uint32_t rows = slab_base + b * kFuSlab + nh * (kFuUnit / 2) * 128;
        wgmma_fence();
#pragma unroll
        for (int q = 0; q < 4; ++q) {                           // stage q = (K-half q>>1, weight hi/lo q&1)
          const int khq = q >> 1;
          const uint64_t wdesc = gmma_desc_sw128(w_base + q * 16384);
          const uint64_t yh = gmma_desc_sw128(rows + khq * kFuRegion);
          const uint64_t yl = gmma_desc_sw128(rows + (2 + khq) * kFuRegion);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            wgmma_f16_n48(d, wdesc + kk * 2, yh + kk * 2, (q == 0 && kk == 0) ? 0u : 1u);
            if ((q & 1) == 0) wgmma_f16_n48(d, wdesc + kk * 2, yl + kk * 2, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (nh == 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&a_empty[b]);
        }
        wgmma_fence_regs(d);
        // pool group j of the half = accumulator columns 8 j .. 8 j + 7 = registers 4 j + 2 h + e of the lane quad
#pragma unroll
        for (int j = 0; j < kFuUnit / 2 / kPool; ++j) {
          float m0 = fmaxf(d[4 * j], d[4 * j + 1]), m1 = fmaxf(d[4 * j + 2], d[4 * j + 3]);
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
          const int gg = ((t0 + nh * (kFuUnit / 2)) >> 3) + j;
          if ((lane & 3) == 0 && gg < kPooled) {
            float* qrow = p.q_out + (static_cast<size_t>(w) * kPooled + gg) * kC;
            qrow[ch0] = m0 * oscale;
            qrow[ch0 + 8] = m1 * oscale;
          }
        }
      }
    }
  }
}

}  // namespace gnm
