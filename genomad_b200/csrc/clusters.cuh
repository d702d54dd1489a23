// Greedy clustering of embeddings at a cosine threshold (gnm_cluster_block, include/gnm.h): one block of rows, in file order.
//
//   nb_mask_kernel     bit i of mask row j = s(j, i) >= thr, for every pair i < j of the block, with s the similarity of
//                      gnm_embedding_neighbours for query j and reference i.  The mainloop is nb_search_kernel's (nb_ring_init,
//                      nb_produce, nb_tile_mma in neighbours.cuh): the same TMA ring and wgmma sequence over the same operand bits,
//                      so the bits are the comparison of the search's own similarities.  Only the epilogue differs: each quad of
//                      lanes ORs its row's fragment bits into 32-column words and stores them.  Reference tiles that hold no
//                      column i < j for any row j of the query tile (above the diagonal) are skipped.
//   cl_resolve_kernel  one CTA: for j ascending, j is a representative iff it is not covered by an earlier block's
//                      representative and no mask bit (j, i) has i a representative of this block.  The 8 warps stage 32 mask rows
//                      at a time in shared memory; warp 0 decides them in order, holding the block's representative bitmap in
//                      registers (lane L: words L + 32 q).
//   cl_probe_filter_kernel  (gnm_cluster_block_probed, between the two) clears mask bit (j, i) unless row i's home list is one of
//                      row j's probes, so row j is compared only with the representatives its probed lists hold.  One thread per
//                      mask word below the diagonal; only set bits are checked, and at a high threshold few are set.
//
// DESIGN.md, "Embedding clusters".
#pragma once
#include "neighbours.cuh"

namespace gnm {

constexpr int kClMaxBlock = 8192;                     // rows per block: mask [8192][256] words = 8 MB
constexpr int kClMaxWords = kClMaxBlock / 32;
constexpr int kClMaskTiles = 4;                       // reference tiles per mask CTA
constexpr int kClStage = 32;                          // mask rows per shared-memory stage of cl_resolve_kernel
constexpr int kClThreads = 256;
constexpr int kClMaskSmem = kNbStages * kNbStageBytes + 1024 + 64;

struct NbMaskParams {
  uint32_t* mask;           // [n][words]; only words holding a column i < j of row j are written
  int n, words, tiles_per_split;
  float thr;
  DeviceStatus* status;
};

// reference tiles with a column i < j for some row j < n of query tile m0: those starting below the tile's last row
__host__ __device__ inline int nb_mask_tiles(int m0, int n) { return ((m0 + kNbBM < n ? m0 + kNbBM : n) - 1 + kNbBN - 1) / kNbBN; }

__global__ void __launch_bounds__(kNbThreads, 1)
nb_mask_kernel(const __grid_constant__ CUtensorMap tm_q_hi, const __grid_constant__ CUtensorMap tm_q_lo,
               const __grid_constant__ CUtensorMap tm_r_hi, const __grid_constant__ CUtensorMap tm_r_lo, const NbMaskParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kNbStages * kNbStageBytes);
  uint64_t* empty = full + kNbStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * kNbBM, t0 = blockIdx.x * p.tiles_per_split;
  const int nt = min(p.tiles_per_split, nb_mask_tiles(m0, p.n) - t0);
  if (nt <= 0) return;                                                     // the split lies above the diagonal

  if (warp == 0 && lane == 0) nb_ring_init(&tm_q_hi, &tm_q_lo, &tm_r_hi, &tm_r_lo, full, empty);
  __syncthreads();

  if (warp == 0 && lane == 0) {
    nb_produce(&tm_q_hi, &tm_q_lo, &tm_r_hi, &tm_r_lo, smem, full, empty, m0, t0, nt, p.status);
  } else if (warp >= 4) {
    const int g = (warp >> 2) - 1, wq = warp & 3;
    const uint32_t base = smem_u32(smem);
    float d[96];
    for (int tt = 0; tt < nt; ++tt) {
      nb_tile_mma(d, base, full, empty, g, tt, p.status);
      const int c0 = (t0 + tt) * kNbBN;                                    // the tile's first column: a multiple of 32
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m0 + g * 64 + wq * 16 + (lane >> 2) + 8 * h;
#pragma unroll
        for (int w = 0; w < kNbBN / 32; ++w) {
          uint32_t bits = 0;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int b = 8 * jj + 2 * (lane & 3) + e;                    // column c0 + 32 w + b
              if (d[4 * (4 * w + jj) + 2 * h + e] >= p.thr && c0 + 32 * w + b < row) bits |= 1u << b;
            }
          }
          bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
          bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
          const int word = c0 / 32 + w;
          if ((lane & 3) == (w & 3) && row < p.n && word < p.words) p.mask[static_cast<size_t>(row) * p.words + word] = bits;
        }
      }
    }
  }
}

// mask word (j, w) with a column i < j: bit i kept iff home[i] is one of probes[j][0 .. nprobe)
__global__ void __launch_bounds__(256) cl_probe_filter_kernel(uint32_t* __restrict__ mask, int n, int words,
                                                              const int32_t* __restrict__ probes, int nprobe,
                                                              const int32_t* __restrict__ home) {
  const long long x = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (x >= static_cast<long long>(n) * words) return;
  const int j = static_cast<int>(x / words), w = static_cast<int>(x - static_cast<long long>(j) * words);
  if (32 * w >= j) return;                                                 // no column i < j: not written by nb_mask_kernel
  const uint32_t bits = mask[x];
  uint32_t keep = bits;
  for (uint32_t b = bits; b; b &= b - 1) {
    const int i = 32 * w + __ffs(b) - 1, h = home[i];
    bool probed = false;
    for (int q = 0; q < nprobe && !probed; ++q) probed = probes[static_cast<size_t>(j) * nprobe + q] == h;
    if (!probed) keep &= ~(1u << (i & 31));
  }
  if (keep != bits) mask[x] = keep;
}

__global__ void __launch_bounds__(kClThreads, 1)
cl_resolve_kernel(const uint32_t* __restrict__ mask, int n, int words, const uint8_t* __restrict__ covered,
                  int32_t* __restrict__ new_reps, int32_t* __restrict__ n_new) {
  __shared__ uint32_t sm[kClStage][kClMaxWords];
  __shared__ uint8_t cov[kClStage];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t rep[kClMaxWords / 32];                                          // warp 0: the block's representatives so far
#pragma unroll
  for (int q = 0; q < kClMaxWords / 32; ++q) rep[q] = 0;
  int cnt = 0;
  for (int c0 = 0; c0 < n; c0 += kClStage) {
    const int rows = min(kClStage, n - c0);
    for (int x = threadIdx.x; x < rows * words; x += kClThreads) {
      const int r = x / words, w = x - r * words, j = c0 + r;
      if (32 * w < j) sm[r][w] = mask[static_cast<size_t>(j) * words + w];   // words with a column i < j
    }
    if (threadIdx.x < rows) cov[threadIdx.x] = covered[c0 + threadIdx.x];
    __syncthreads();
    if (warp == 0) {
      for (int r = 0; r < rows; ++r) {
        const int j = c0 + r;
        if (cov[r]) continue;
        uint32_t hit = 0;
#pragma unroll
        for (int q = 0; q < kClMaxWords / 32; ++q) {
          const int w = lane + 32 * q;
          if (32 * w < j) hit |= sm[r][w] & rep[q];
        }
        if (__any_sync(0xffffffffu, hit != 0)) continue;
        if (lane == ((j >> 5) & 31)) {
#pragma unroll
          for (int q = 0; q < kClMaxWords / 32; ++q)
            if (q == (j >> 10)) rep[q] |= 1u << (j & 31);
        }
        if (lane == 0) new_reps[cnt] = j;
        ++cnt;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *n_new = cnt;
}

}  // namespace gnm
