// Inverted-list search in the encoder's embedding space (gnm_ivf_search, include/gnm.h): for every query row, the k reference rows
// of highest cosine similarity among the rows of the lists it probes, under the exact search's total order (similarity
// descending, reference index ascending).  The similarities are those of gnm_embedding_neighbours bit for bit: the operands are
// the halves of nb_prep_kernel, the MMA is nb_tile_mma and the admission nb_offer (neighbours.cuh).  Only the decomposition
// of the work is new.
//
//   ivf_keys_kernel     the list each (query, list) pair probes, as a sort key (pairs come in query order; a list outside
//                       [0, lists) or a query outside [0, n_query) gets the key `lists`, sorts last and is dropped).  A
//                       stable radix sort then orders the pairs by (list, query).
//   ivf_lists_kernel    one thread per list: its first sorted pair (a lower bound in the sorted keys), and its work items and
//                       partial lists, whose exclusive sums give every item and partial list its place.
//   ivf_gather_kernel   one warp per sorted pair: the query's row copied to the pair's row of a contiguous buffer, whose halves
//                       nb_prep_kernel makes, so a list's queries are consecutive rows one TMA map reads; and the column of the
//                       query's own row in the list.
//   ivf_search_kernel   persistent CTAs of nb_search_kernel's shape, each taking work items round robin.  An item is (list l,
//                       a tile of <= 128 of l's pairs, a range of <= kIvfItemTiles of l's 192-row reference tiles); its
//                       reference tiles start at any row, and the epilogue drops columns outside l's rows and rows outside the
//                       item's pairs.  Every item writes one sorted partial list per pair.
//   ivf_merge_kernel    one warp per query: the partial lists of all its pairs merged (nb_merge_warp), columns mapped to global
//                       reference indices.
//                       Keys are distinct, so the order of the merges does not matter.
// The reference halves come from nb_prep_kernel once per reference chunk (gnm_ivf_prepare), not once per call.
//
// Growing lists (gnm_ivf_search_ranges): list l holds only the prefix [off[l], end[l]) of its slots [off[l], off[l + 1]).  The
// list-reading code is instantiated with kGrow = true, which reads end[l] where the index path reads off[l + 1]; `off` then holds
// the lists + 1 slot offsets followed by the lists ends (ivf_ends_kernel).  Keys, gather and halves are shared.
//
// DESIGN.md, "Embedding index".
#pragma once
#include "neighbours.cuh"

namespace gnm {

constexpr int kIvfItemTiles = 8;      // reference tiles per work item at most: a long list is cut into ranges of 1,536 rows
constexpr int kIvfMaxProbe = 64;

// reference tile ranges of a list of `rows` rows (0 for an empty list)
__host__ __device__ __forceinline__ long long ivf_ranges(long long rows) {
  const long long tiles = (rows + kNbBN - 1) / kNbBN;
  return (tiles + kIvfItemTiles - 1) / kIvfItemTiles;
}

// the end of list l's rows: off[l + 1], or with kGrow its live prefix's end, stored after the lists + 1 offsets
template <bool kGrow>
__device__ __forceinline__ long long ivf_end(const long long* __restrict__ off, int l, int lists) {
  return kGrow ? off[lists + 1 + l] : off[l + 1];
}

__global__ void __launch_bounds__(256) ivf_keys_kernel(const int32_t* __restrict__ pair_query, const int32_t* __restrict__ pair_list,
                                                       int n_pairs, int n_query, int lists, uint32_t* __restrict__ keys,
                                                       int32_t* __restrict__ vals) {
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= n_pairs) return;
  const int l = pair_list[e], q = pair_query[e];
  keys[e] = (l >= 0 && l < lists && q >= 0 && q < n_query) ? static_cast<uint32_t>(l) : static_cast<uint32_t>(lists);
  vals[e] = e;
}

__device__ __forceinline__ int ivf_lower_bound(const uint32_t* __restrict__ a, int n, uint32_t x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// l in [0, lists]: pstart[l] = first sorted pair of list l (pstart[lists] = the pairs that probe a list of this call);
// items[l] = ceil(pairs / 128) x ranges, parts[l] = pairs x ranges (0 at l = lists, so their exclusive sums end in the totals)
template <bool kGrow>
__device__ __forceinline__ void ivf_lists(const uint32_t* __restrict__ skeys, int n_pairs, const long long* __restrict__ off, int lists,
                                          int* __restrict__ pstart, long long* __restrict__ items, long long* __restrict__ parts) {
  const int l = blockIdx.x * 256 + threadIdx.x;
  if (l > lists) return;
  const int a = ivf_lower_bound(skeys, n_pairs, static_cast<uint32_t>(l));
  pstart[l] = a;
  if (l == lists) { items[l] = 0; parts[l] = 0; return; }
  const long long cnt = ivf_lower_bound(skeys, n_pairs, static_cast<uint32_t>(l) + 1) - a;
  const long long nr = ivf_ranges(ivf_end<kGrow>(off, l, lists) - off[l]);
  items[l] = (cnt + kNbBM - 1) / kNbBM * nr;
  parts[l] = cnt * nr;
}

__global__ void __launch_bounds__(256) ivf_lists_kernel(const uint32_t* __restrict__ skeys, int n_pairs,
                                                        const long long* __restrict__ off, int lists, int* __restrict__ pstart,
                                                        long long* __restrict__ items, long long* __restrict__ parts) {
  ivf_lists<false>(skeys, n_pairs, off, lists, pstart, items, parts);
}

__global__ void __launch_bounds__(256) ivf_grow_lists_kernel(const uint32_t* __restrict__ skeys, int n_pairs,
                                                             const long long* __restrict__ off, int lists, int* __restrict__ pstart,
                                                             long long* __restrict__ items, long long* __restrict__ parts) {
  ivf_lists<true>(skeys, n_pairs, off, lists, pstart, items, parts);
}

// off[lists + 1 + l] = end[l] clamped to list l's slots [off[l], off[l + 1]]
__global__ void __launch_bounds__(256) ivf_ends_kernel(const long long* __restrict__ end, int lists, long long* __restrict__ off) {
  const int l = blockIdx.x * 256 + threadIdx.x;
  if (l < lists) off[lists + 1 + l] = min(max(end[l], off[l]), off[l + 1]);
}

// one warp per sorted pair p: its query's fp32 row -> row p of g_raw (zeros for a dropped pair), whose halves nb_prep_kernel
// then makes row by row; slot_of[pair] = p (-1 for a dropped pair); self_col[p] = the row of list l holding global index
// self_index0 + q (rows of a list ascend in global index), else -1
__global__ void __launch_bounds__(256) ivf_gather_kernel(const float* __restrict__ query, const int32_t* __restrict__ pair_query,
                                                         const uint32_t* __restrict__ skeys, const int32_t* __restrict__ svals,
                                                         int n_pairs, const int* __restrict__ pstart, int lists,
                                                         const long long* __restrict__ off, const long long* __restrict__ ref_index,
                                                         long long self_index0, float* __restrict__ g_raw, int* __restrict__ slot_of,
                                                         int* __restrict__ self_col) {
  const int p = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= n_pairs) return;
  const int e = svals[p];
  float4* d = reinterpret_cast<float4*>(g_raw + static_cast<size_t>(p) * kNbDim);
  if (p >= pstart[lists]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) d[lane + 32 * i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane == 0) { slot_of[e] = -1; self_col[p] = -1; }
    return;
  }
  const int q = pair_query[e];
  const float4* src = reinterpret_cast<const float4*>(query + static_cast<size_t>(q) * kNbDim);
#pragma unroll
  for (int i = 0; i < 4; ++i) d[lane + 32 * i] = src[lane + 32 * i];
  if (lane == 0) {
    slot_of[e] = p;
    int col = -1;
    if (self_index0 >= 0) {
      const long long g = self_index0 + q;
      const int l = static_cast<int>(skeys[p]);
      long long lo = off[l], hi = off[l + 1];
      while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (ref_index[mid] < g) lo = mid + 1; else hi = mid;
      }
      if (lo < off[l + 1] && ref_index[lo] == g) col = static_cast<int>(lo);
    }
    self_col[p] = col;
  }
}

struct IvfSearchParams {
  float* part_sim;               // [partial lists][k], each sorted
  int32_t* part_idx;             // reference rows of this call, -1 = empty
  const long long* off;          // [lists + 1] rows of list l: [off[l], off[l + 1])
  const int* pstart;             // [lists + 1]
  const long long* ibase;        // [lists + 1] first item of list l; ibase[lists] = items
  const long long* pbase;        // [lists + 1] first partial list of list l
  const int* self_col;           // [pairs]
  int lists, k;
  DeviceStatus* status;
};

// one work item, decoded the same way by every thread of the CTA
struct IvfItem {
  int m0, nq;                    // its pairs: sorted rows m0 .. m0 + nq - 1 of the gathered queries
  int r0, nt, hi;                // reference tiles at rows r0, r0 + 192, ... (nt of them); columns >= hi belong to later lists
  long long part0;               // partial list of its first pair; pair m0 + i writes part0 + i
};

template <bool kGrow>
__device__ __forceinline__ IvfItem ivf_item(const IvfSearchParams& p, long long i) {
  int lo = 0, hi = p.lists;                      // the last l with ibase[l] <= i (empty lists share their successor's base)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.ibase[mid] <= i) lo = mid; else hi = mid - 1;
  }
  const int l = lo;
  const long long rows = (kGrow ? p.off[p.lists + 1 + l] : p.off[l + 1]) - p.off[l], nr = ivf_ranges(rows), loc = i - p.ibase[l];
  const long long u = loc / nr, r = loc % nr;
  const int cnt = p.pstart[l + 1] - p.pstart[l];
  IvfItem it;
  it.m0 = p.pstart[l] + static_cast<int>(u) * kNbBM;
  it.nq = min(kNbBM, cnt - static_cast<int>(u) * kNbBM);
  const int t0 = static_cast<int>(r) * kIvfItemTiles;
  it.nt = min(kIvfItemTiles, static_cast<int>((rows + kNbBN - 1) / kNbBN) - t0);
  it.r0 = static_cast<int>(p.off[l]) + t0 * kNbBN;
  it.hi = static_cast<int>(kGrow ? p.off[p.lists + 1 + l] : p.off[l + 1]);
  it.part0 = p.pbase[l] + r * cnt + static_cast<long long>(u) * kNbBM;
  return it;
}

// TMA producer of one item: gathered query tile m0 against the reference tiles at rows r0 + 192 t, t < nt, K chunks ascending;
// it0 = the ring position of its first load (the CTA's loads so far)
__device__ __forceinline__ void ivf_produce(const CUtensorMap* tm_q_hi, const CUtensorMap* tm_q_lo, const CUtensorMap* tm_r_hi,
                                            const CUtensorMap* tm_r_lo, uint8_t* smem, uint64_t* full, uint64_t* empty, int m0,
                                            int r0, int nt, int it0, DeviceStatus* status) {
  const uint64_t pol = l2_policy_evict_last();
  for (int j = 0; j < nt * kNbChunks; ++j) {
    const int it = it0 + j;
    const int s = it % kNbStages;
    const uint32_t ph = (it / kNbStages) & 1;
    mbar_wait(&empty[s], ph ^ 1, status, 700 + s);
    mbar_arrive_expect_tx(&full[s], kNbStageBytes);
    uint8_t* st = smem + s * kNbStageBytes;
    const int k0 = (j % kNbChunks) * kNbBK, rr = r0 + (j / kNbChunks) * kNbBN;
    tma_load_2d_hint(st, tm_q_hi, &full[s], k0, m0, pol);
    tma_load_2d_hint(st + kNbATile, tm_q_lo, &full[s], k0, m0, pol);
    tma_load_2d_hint(st + 2 * kNbATile, tm_r_hi, &full[s], k0, rr, pol);
    tma_load_2d_hint(st + 2 * kNbATile + kNbBTile, tm_r_lo, &full[s], k0, rr, pol);
  }
}

__global__ void __launch_bounds__(kNbThreads, 1)
ivf_search_kernel(const __grid_constant__ CUtensorMap tm_q_hi, const __grid_constant__ CUtensorMap tm_q_lo,
                  const __grid_constant__ CUtensorMap tm_r_hi, const __grid_constant__ CUtensorMap tm_r_lo, const IvfSearchParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int k = p.k;
  float* lsim = reinterpret_cast<float*>(smem + kNbStages * kNbStageBytes);     // [128 queries][k]
  int* lidx = reinterpret_cast<int*>(lsim + kNbBM * k);
  uint64_t* full = reinterpret_cast<uint64_t*>(lidx + kNbBM * k);
  uint64_t* empty = full + kNbStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_items = p.ibase[p.lists];
  if (warp == 0 && lane == 0) nb_ring_init(&tm_q_hi, &tm_q_lo, &tm_r_hi, &tm_r_lo, full, empty);
  __syncthreads();

  if (warp == 0 && lane == 0) {
    // ===================================================================== TMA producer
    int it0 = 0;
    for (long long i = blockIdx.x; i < n_items; i += gridDim.x) {
      const IvfItem w = ivf_item<false>(p, i);
      ivf_produce(&tm_q_hi, &tm_q_lo, &tm_r_hi, &tm_r_lo, smem, full, empty, w.m0, w.r0, w.nt, it0, p.status);
      it0 += w.nt * kNbChunks;
    }
  } else if (warp >= 4) {
    // ===================================================================== MMA + top-k: warpgroup g owns tile rows 64 g .. 64 g + 63
    const int g = (warp >> 2) - 1, wq = warp & 3;
    const uint32_t base = smem_u32(smem);
    int rowl[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) rowl[h] = g * 64 + wq * 16 + (lane >> 2) + 8 * h;
    int tg = 0;                                                   // the CTA's tiles so far: the ring position
    float d[96];
    for (long long i = blockIdx.x; i < n_items; i += gridDim.x) {
      const IvfItem w = ivf_item<false>(p, i);
      int self_col[2], wi[2], wp[2];
      float ws[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const bool mine = rowl[h] < w.nq;
        self_col[h] = mine ? p.self_col[w.m0 + rowl[h]] : -1;
        ws[h] = mine ? -CUDART_INF_F : CUDART_INF_F;             // +inf: a row outside the item admits nothing
        wi[h] = -1; wp[h] = k - 1;
        for (int a = lane & 3; a < k; a += 4) { lsim[rowl[h] * k + a] = -CUDART_INF_F; lidx[rowl[h] * k + a] = -1; }
      }
      __syncwarp();
      for (int tt = 0; tt < w.nt; ++tt, ++tg) {
        nb_tile_mma(d, base, full, empty, g, tg, p.status);
        const int n0 = w.r0 + tt * kNbBN + 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int j = 0; j < kNbBN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float v = d[4 * j + 2 * h + e];
              if (__any_sync(0xffffffffu, v >= ws[h]))
                nb_offer(v, n0 + 8 * j + e, rowl[h], self_col[h], w.hi, k, ws[h], wi[h], wp[h], lsim, lidx);
            }
          }
        }
      }
      __syncwarp();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (rowl[h] >= w.nq) continue;
        const float* rs = lsim + rowl[h] * k;
        const int* ri = lidx + rowl[h] * k;
        const size_t o = static_cast<size_t>(w.part0 + rowl[h]) * k;
        for (int a = lane & 3; a < k; a += 4) {
          const float s = rs[a]; const int x = ri[a];
          int rank = 0;
          for (int b = 0; b < k; ++b) rank += nb_beats(rs[b], ri[b], s, x) || (b < a && rs[b] == s && ri[b] == x);
          p.part_sim[o + rank] = s;
          p.part_idx[o + rank] = x;
        }
      }
      __syncwarp();
    }
  }
}

// ivf_search_kernel over growing lists (kGrow).  Its body repeats ivf_search_kernel's, which stays as written before so that the
// index search keeps the exact code it was validated with (tools/sass_diff.py).
__global__ void __launch_bounds__(kNbThreads, 1)
ivf_grow_search_kernel(const __grid_constant__ CUtensorMap tm_q_hi, const __grid_constant__ CUtensorMap tm_q_lo,
                       const __grid_constant__ CUtensorMap tm_r_hi, const __grid_constant__ CUtensorMap tm_r_lo,
                       const IvfSearchParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int k = p.k;
  float* lsim = reinterpret_cast<float*>(smem + kNbStages * kNbStageBytes);     // [128 queries][k]
  int* lidx = reinterpret_cast<int*>(lsim + kNbBM * k);
  uint64_t* full = reinterpret_cast<uint64_t*>(lidx + kNbBM * k);
  uint64_t* empty = full + kNbStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_items = p.ibase[p.lists];
  if (warp == 0 && lane == 0) nb_ring_init(&tm_q_hi, &tm_q_lo, &tm_r_hi, &tm_r_lo, full, empty);
  __syncthreads();

  if (warp == 0 && lane == 0) {
    // ===================================================================== TMA producer
    int it0 = 0;
    for (long long i = blockIdx.x; i < n_items; i += gridDim.x) {
      const IvfItem w = ivf_item<true>(p, i);
      ivf_produce(&tm_q_hi, &tm_q_lo, &tm_r_hi, &tm_r_lo, smem, full, empty, w.m0, w.r0, w.nt, it0, p.status);
      it0 += w.nt * kNbChunks;
    }
  } else if (warp >= 4) {
    // ===================================================================== MMA + top-k: warpgroup g owns tile rows 64 g .. 64 g + 63
    const int g = (warp >> 2) - 1, wq = warp & 3;
    const uint32_t base = smem_u32(smem);
    int rowl[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) rowl[h] = g * 64 + wq * 16 + (lane >> 2) + 8 * h;
    int tg = 0;                                                   // the CTA's tiles so far: the ring position
    float d[96];
    for (long long i = blockIdx.x; i < n_items; i += gridDim.x) {
      const IvfItem w = ivf_item<true>(p, i);
      int self_col[2], wi[2], wp[2];
      float ws[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const bool mine = rowl[h] < w.nq;
        self_col[h] = mine ? p.self_col[w.m0 + rowl[h]] : -1;
        ws[h] = mine ? -CUDART_INF_F : CUDART_INF_F;             // +inf: a row outside the item admits nothing
        wi[h] = -1; wp[h] = k - 1;
        for (int a = lane & 3; a < k; a += 4) { lsim[rowl[h] * k + a] = -CUDART_INF_F; lidx[rowl[h] * k + a] = -1; }
      }
      __syncwarp();
      for (int tt = 0; tt < w.nt; ++tt, ++tg) {
        nb_tile_mma(d, base, full, empty, g, tg, p.status);
        const int n0 = w.r0 + tt * kNbBN + 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int j = 0; j < kNbBN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float v = d[4 * j + 2 * h + e];
              if (__any_sync(0xffffffffu, v >= ws[h]))
                nb_offer(v, n0 + 8 * j + e, rowl[h], self_col[h], w.hi, k, ws[h], wi[h], wp[h], lsim, lidx);
            }
          }
        }
      }
      __syncwarp();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (rowl[h] >= w.nq) continue;
        const float* rs = lsim + rowl[h] * k;
        const int* ri = lidx + rowl[h] * k;
        const size_t o = static_cast<size_t>(w.part0 + rowl[h]) * k;
        for (int a = lane & 3; a < k; a += 4) {
          const float s = rs[a]; const int x = ri[a];
          int rank = 0;
          for (int b = 0; b < k; ++b) rank += nb_beats(rs[b], ri[b], s, x) || (b < a && rs[b] == s && ri[b] == x);
          p.part_sim[o + rank] = s;
          p.part_idx[o + rank] = x;
        }
      }
      __syncwarp();
    }
  }
}

// one warp per query: the partial lists of its pairs (pair_query ascending: a binary search finds them) merged; reference rows
// -> ref_index[row]
template <bool kGrow>
__device__ __forceinline__ void ivf_merge(const float* __restrict__ part_sim, const int32_t* __restrict__ part_idx,
                                          const int32_t* __restrict__ pair_query, const int32_t* __restrict__ pair_list, int n_pairs,
                                          const int* __restrict__ slot_of, const long long* __restrict__ off, int lists,
                                          const int* __restrict__ pstart, const long long* __restrict__ pbase, int n_query, int k,
                                          const long long* __restrict__ ref_index, float* out_sim, long long* out_idx) {
  __shared__ float ms[8][kNbMaxK];
  __shared__ long long mi[8][kNbMaxK];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * 8 + w;
  if (q >= n_query) return;
  int e0 = 0, hi = n_pairs;
  while (e0 < hi) {
    const int mid = (e0 + hi) >> 1;
    if (pair_query[mid] < q) e0 = mid + 1; else hi = mid;
  }
  float as[2] = {-CUDART_INF_F, -CUDART_INF_F};
  long long ai[2] = {-1, -1};
  for (int e = e0; e < n_pairs && pair_query[e] == q; ++e) {
    const int sp = slot_of[e];
    if (sp < 0) continue;
    const int l = pair_list[e];
    const long long nr = ivf_ranges(ivf_end<kGrow>(off, l, lists) - off[l]), cnt = pstart[l + 1] - pstart[l];
    for (long long r = 0; r < nr; ++r) {
      const size_t o = static_cast<size_t>(pbase[l] + r * cnt + (sp - pstart[l])) * k;
      float bs[2] = {-CUDART_INF_F, -CUDART_INF_F};
      long long bi[2] = {-1, -1};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int x = lane + 32 * h;
        if (x < k) {
          const int i = part_idx[o + x];
          bs[h] = i < 0 ? -CUDART_INF_F : part_sim[o + x];
          bi[h] = i < 0 ? -1 : ref_index[i];
        }
      }
      nb_merge_warp(as, ai, bs, bi, k, ms[w], mi[w]);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int x = lane + 32 * h;
    if (x < k) { out_sim[static_cast<size_t>(q) * k + x] = as[h]; out_idx[static_cast<size_t>(q) * k + x] = ai[h]; }
  }
}

__global__ void __launch_bounds__(256) ivf_merge_kernel(const float* __restrict__ part_sim, const int32_t* __restrict__ part_idx,
                                                        const int32_t* __restrict__ pair_query, const int32_t* __restrict__ pair_list,
                                                        int n_pairs, const int* __restrict__ slot_of, const long long* __restrict__ off,
                                                        const int* __restrict__ pstart, const long long* __restrict__ pbase,
                                                        int n_query, int k, const long long* __restrict__ ref_index, float* out_sim,
                                                        long long* out_idx) {
  ivf_merge<false>(part_sim, part_idx, pair_query, pair_list, n_pairs, slot_of, off, 0, pstart, pbase, n_query, k, ref_index, out_sim,
                   out_idx);
}

__global__ void __launch_bounds__(256) ivf_grow_merge_kernel(const float* __restrict__ part_sim, const int32_t* __restrict__ part_idx,
                                                             const int32_t* __restrict__ pair_query,
                                                             const int32_t* __restrict__ pair_list, int n_pairs,
                                                             const int* __restrict__ slot_of, const long long* __restrict__ off,
                                                             int lists, const int* __restrict__ pstart,
                                                             const long long* __restrict__ pbase, int n_query, int k,
                                                             const long long* __restrict__ ref_index, float* out_sim, long long* out_idx) {
  ivf_merge<true>(part_sim, part_idx, pair_query, pair_list, n_pairs, slot_of, off, lists, pstart, pbase, n_query, k, ref_index,
                  out_sim, out_idx);
}

}  // namespace gnm
