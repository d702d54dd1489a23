// K5 on the tensor cores: attention logits = mpi @ w_qk  (reference genomad/neural_network/igloo.py:211), [n x 2100] x [2100 x 749],
// and (round 2) the two Dense(512) projections of the head (reference genomad/neural_network/model.py:28, 40): the same
// kernel with K = 256 / 512 and N = 512; bias + BatchNorm + ReLU are applied by splitk_reduce_epi_kernel (dense.cuh).
//
// fp32 semantics on the tensor cores: both operands are split into two TF32 halves, x = hi + lo with hi = x with the low 13
// mantissa bits cleared and lo = (x - hi) likewise truncated (so the hardware's fp32 -> tf32 conversion has nothing left to
// round), and D = Ahi*Bhi + Alo*Bhi + Ahi*Blo accumulates in one fp32 accumulator (the dropped lo*lo term and the truncation of
// lo are ~2^-20 relative; TF32 keeps fp32's 8-bit exponent, so the ~1e-32 weights of the shipped model need no scaling).
// The split halves are written where the operands are produced (patch_finish_kernel for mpi, gnm_create for w_qk^T), TMA
// brings them in as 128-byte-swizzled K-major tiles, and two consumer warpgroups (64 rows of the 128-row tile each) issue 12
// wgmma (M64 N256 K8, tf32) per 32-wide K chunk into register accumulators.
//
// grid = (3 N tiles of 256 columns, ceil(n/128) M tiles, kLgSplits K splits): 144 CTAs at batch 1024.  Each split writes its
// partial product to part[z][m][752]; splitk_reduce_kernel adds the partials in fixed order, so a window's logits do not
// depend on the batch it is in.
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace gnm {

constexpr int kLgBM = 128, kLgBN = 256, kLgBK = 32;               // fp32 elements; one K chunk = 128 bytes per row
constexpr int kLgSplits = 6;
constexpr int kLgChunks = (kPatches + kLgBK - 1) / kLgBK;         // 66 (the last one is partly out of bounds -> zero filled)
constexpr int kLgChunksPerSplit = kLgChunks / kLgSplits;          // 11
static_assert(kLgChunksPerSplit * kLgSplits == kLgChunks, "K chunks must divide evenly among the splits");
constexpr int kLgStages = 2;
constexpr int kLgATile = kLgBM * 128, kLgBTile = kLgBN * 128;     // 16 KB, 32 KB
constexpr int kLgStageBytes = 2 * kLgATile + 2 * kLgBTile;        // A hi | A lo | B hi | B lo = 96 KB
constexpr int kLgSmem = kLgStages * kLgStageBytes + 1024 + 256;
constexpr int kLgThreads = 384;                                   // warpgroup 0: TMA thread; warpgroups 1, 2: MMA + epilogue

struct LogitsTcParams {
  float* part;               // [gridDim.z splits][n_rows][ldc]
  int ldc;                   // 752 (logits) / 512 (dense)
  int n_rows;                // windows in this step
  int n_cols;                // 749 / 512
  int chunks_total;          // K chunks of 32 fp32 (the last one may be partly out of bounds -> zero filled by TMA)
  int chunks_per_split;      // gridDim.z * chunks_per_split >= chunks_total, every split owns >= 1 chunk
  DeviceStatus* status;
};

// x = hi + lo, both exactly representable as TF32 (low 13 mantissa bits zero)
__host__ __device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
#ifdef __CUDA_ARCH__
  hi = __uint_as_float(__float_as_uint(x) & 0xffffe000u);
  lo = __uint_as_float(__float_as_uint(x - hi) & 0xffffe000u);
#else
  uint32_t u; memcpy(&u, &x, 4); u &= 0xffffe000u; memcpy(&hi, &u, 4);
  float r = x - hi; memcpy(&u, &r, 4); u &= 0xffffe000u; memcpy(&lo, &u, 4);
#endif
}

__global__ void __launch_bounds__(kLgThreads, 1)
logits_tc_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                 const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                 const LogitsTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kLgStages * kLgStageBytes);
  uint64_t* full = bars;              // [2]
  uint64_t* empty = bars + 2;         // [2]  one arrival per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * kLgBN, m0 = blockIdx.y * kLgBM, z = blockIdx.z;
  const int c0 = z * p.chunks_per_split;
  const int nc = min(p.chunks_per_split, p.chunks_total - c0);     // >= 1 by construction of the grid

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_a_hi); tma_prefetch_desc(&tm_a_lo); tma_prefetch_desc(&tm_b_hi); tma_prefetch_desc(&tm_b_lo);
    for (int i = 0; i < kLgStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0 && lane == 0) {
    // ===================================================================== TMA producer
    const uint64_t pol_a = l2_policy_evict_first(), pol_b = l2_policy_evict_last();     // w_qk is re-read by every M tile
    for (int c = 0; c < nc; ++c) {
      const int s = c % kLgStages;
      const uint32_t ph = (c / kLgStages) & 1;
      mbar_wait(&empty[s], ph ^ 1, p.status, 500 + s);
      mbar_arrive_expect_tx(&full[s], kLgStageBytes);
      uint8_t* st = smem + s * kLgStageBytes;
      const int k0 = (c0 + c) * kLgBK;
      tma_load_2d_hint(st, &tm_a_hi, &full[s], k0, m0, pol_a);
      tma_load_2d_hint(st + kLgATile, &tm_a_lo, &full[s], k0, m0, pol_a);
      tma_load_2d_hint(st + 2 * kLgATile, &tm_b_hi, &full[s], k0, n0, pol_b);
      tma_load_2d_hint(st + 2 * kLgATile + kLgBTile, &tm_b_lo, &full[s], k0, n0, pol_b);
    }
  } else if (warp >= 4) {
    // ===================================================================== MMA + epilogue: warpgroup g owns rows 64 g .. 64 g + 63
    const int g = (warp >> 2) - 1, wq = warp & 3;
    const uint32_t base = smem_u32(smem);
    float d[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0.f;
    for (int c = 0; c < nc; ++c) {
      const int s = c % kLgStages;
      const uint32_t ph = (c / kLgStages) & 1;
      mbar_wait(&full[s], ph, p.status, 510 + s);
      const uint32_t st = base + s * kLgStageBytes;
      const uint64_t a_hi = gmma_desc_sw128(st + g * 64 * 128), a_lo = gmma_desc_sw128(st + kLgATile + g * 64 * 128);
      const uint64_t b_hi = gmma_desc_sw128(st + 2 * kLgATile), b_lo = gmma_desc_sw128(st + 2 * kLgATile + kLgBTile);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kLgBK / 8; ++kk) {                   // K = 8 TF32 = 32 bytes per instruction
        wgmma_tf32_n256(d, a_hi + kk * 2, b_hi + kk * 2, (c == 0 && kk == 0) ? 0u : 1u);
        wgmma_tf32_n256(d, a_lo + kk * 2, b_hi + kk * 2, 1u);
        wgmma_tf32_n256(d, a_hi + kk * 2, b_lo + kk * 2, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);                       // the stage may be refilled
    }
    wgmma_fence_regs(d);
    // ===================================================================== epilogue: rows = windows, columns = logits
    const int r0 = m0 + g * 64 + wq * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = r0 + 8 * h;
      if (m >= p.n_rows) continue;
      float* dst = p.part + (static_cast<size_t>(z) * p.n_rows + m) * p.ldc;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int col = n0 + 8 * j + 2 * (lane & 3);
        const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
        if (col + 1 < p.n_cols) *reinterpret_cast<float2*>(dst + col) = make_float2(v0, v1);
        else if (col < p.n_cols) dst[col] = v0;
      }
    }
  }
}

}  // namespace gnm
