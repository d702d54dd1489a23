// Contig sequence bytes -> the windows of the nn-classification path, on the device.
//
// Reference semantics (the same rules csrc/fasta.cpp applies to FASTA text; both must agree byte for byte):
//   read_fasta(strip_n=True)   genomad/sequence.py:96-121   leading / trailing 'n'/'N' of the whole contig are stripped; a
//                              contig that is then empty has no window (the reference drops it)
//   seq_windows(6000, 2500)    genomad/sequence.py:150-167  consecutive 6000-nt slices of the stripped contig; a shorter last
//                              slice is kept only if it has >= 2500 nt, except that the first is always kept; at most one
//                              with --single-window
//   N rule / pad / upper-case  genomad/modules/nn_classification.py:70-72   a window other than the first is skipped if its
//                              RAW bytes hold more than 4000 'N' (case-sensitive: 'n' does not count); windows are
//                              ASCII-upper-cased and right-padded with 'N' to 6000 bytes
//
// Planning is two passes of contig_plan_kernel (one CTA per contig) around contig_scan_kernel, and needs no scratch memory:
//   count  : strip, candidate windows, N rule -> kept windows per contig, written into the caller's offsets array;
//   scan   : counts -> CSR offsets in place; the total (or an error code) lands in offsets[n_contigs], which the host reads;
//   write  : only once the host has checked the total against the caller's capacity: each contig writes its kept windows'
//            starts and lengths at its offset.  A contig whose candidates were all kept (almost all of them) skips the N
//            counts the second time, so the pass re-reads little beyond the stripped ends.
// gather_windows_kernel then turns (start, length) pairs into the uint8 [n][6000] rows that gnm_forward_ascii takes.
#pragma once
#include "common.cuh"

namespace gnm {

constexpr int kMinTail = 2500;                       // shortest kept last window     (nn_classification.py:68)
constexpr int kMaxN = 4000;                          // N rule                          (nn_classification.py:70)
constexpr int kPlanThreads = 256;
constexpr int kPlanWarps = kPlanThreads / 32;
constexpr int kScanThreads = 1024;
constexpr int kScanPer = 4;                          // counts per thread and round of contig_scan_kernel
constexpr int kGatherThreads = 128;
constexpr int32_t kPlanOverflow = -1;                // offsets[n_contigs] after the scan: more than INT32_MAX windows
constexpr int32_t kPlanBadOffsets = -2;              //   ... a contig's end lies before its start
constexpr int32_t kCountOverflow = INT32_MIN;        // count pass: this contig alone has more than INT32_MAX windows

// 0xff in every byte of a 32-bit word (whose first byte has index `base`) that lies inside [a, b)
__device__ __forceinline__ uint32_t byte_range_mask(int64_t base, int64_t a, int64_t b) {
  const int64_t s = a - base, e = b - base;
  const uint32_t lo = s <= 0 ? 0xffffffffu : s >= 4 ? 0u : 0xffffffffu << (8 * s);
  const uint32_t hi = e >= 4 ? 0xffffffffu : e <= 0 ? 0u : 0xffffffffu >> (32 - 8 * e);
  return lo & hi;
}
__device__ __forceinline__ uint32_t word_of(const uint4& v, int k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }

// 16-byte vectors covering [a, b) of seq, from the aligned vector that holds byte a: every vector holds at least one byte of the
// range, so no load leaves the pages of the caller's buffer.  first = the vector's first byte index (may be below a).
struct VecSpan {
  const uint4* v0; int64_t first; int64_t n;
  __device__ __forceinline__ VecSpan(const uint8_t* seq, int64_t a, int64_t b) {
    const uintptr_t pa = reinterpret_cast<uintptr_t>(seq + a) & ~uintptr_t(15);
    const uintptr_t pb = (reinterpret_cast<uintptr_t>(seq + b) + 15) & ~uintptr_t(15);
    v0 = reinterpret_cast<const uint4*>(pa);
    first = a - static_cast<int64_t>(reinterpret_cast<uintptr_t>(seq + a) - pa);
    n = b > a ? static_cast<int64_t>((pb - pa) / 16) : 0;
  }
};

// 0xff per byte that is neither 'n' nor 'N' ('N' | 0x20 == 'n', and no other byte maps there)
__device__ __forceinline__ uint32_t not_n_bytes(uint32_t w) { return __vcmpne4(w | 0x20202020u, 0x6e6e6e6eu); }

// First (kLast = false) or last (kLast = true) index in [a, b) whose byte is not 'n'/'N', or -1.  The whole CTA scans 16 bytes
// per thread and round, from the end it starts at, and stops after the first round that finds one: a contig that does not start
// with a run of N costs one round; an all-N contig is read once.
template <bool kLast>
__device__ int64_t block_find_non_n(const uint8_t* __restrict__ seq, int64_t a, int64_t b, unsigned long long* s_best) {
  const VecSpan sp(seq, a, b);
  if (threadIdx.x == 0) *s_best = kLast ? 0ull : ~0ull;
  __syncthreads();
  for (int64_t r0 = 0; r0 < sp.n; r0 += blockDim.x) {
    const int64_t j = r0 + threadIdx.x;
    int64_t hit = -1;
    if (j < sp.n) {
      const int64_t jv = kLast ? sp.n - 1 - j : j;
      const uint4 v = sp.v0[jv];
      const int64_t base = sp.first + 16 * jv;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int k = kLast ? 3 - q : q;
        const uint32_t m = not_n_bytes(word_of(v, k)) & byte_range_mask(base + 4 * k, a, b);
        if (m && hit < 0) hit = base + 4 * k + (kLast ? (31 - __clz(m)) / 8 : (__ffs(m) - 1) / 8);
      }
    }
    if (__syncthreads_or(hit >= 0)) {
      if (hit >= 0) {
        if (kLast) atomicMax(s_best, static_cast<unsigned long long>(hit));
        else atomicMin(s_best, static_cast<unsigned long long>(hit));
      }
      __syncthreads();
      const int64_t res = static_cast<int64_t>(*s_best);
      __syncthreads();                                   // every thread has read s_best before a later call resets it
      return res;
    }
  }
  return -1;
}

// 'N' bytes (upper case only) in [a, b), summed over the warp
__device__ __forceinline__ int warp_count_N(const uint8_t* __restrict__ seq, int64_t a, int64_t b) {
  const VecSpan sp(seq, a, b);
  const int lane = threadIdx.x & 31;
  int n = 0;
  for (int64_t j = lane; j < sp.n; j += 32) {
    const uint4 v = sp.v0[j];
    const int64_t base = sp.first + 16 * j;
    const bool edge = base < a || base + 16 > b;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t m = __vcmpeq4(word_of(v, k), 0x4e4e4e4eu);
      if (edge) m &= byte_range_mask(base + 4 * k, a, b);
      n += __popc(m) >> 3;
    }
  }
  return __reduce_add_sync(0xffffffffu, n);
}

// Candidate windows of a stripped contig of L > 0 nt at window step s (1 <= s <= 6000): candidate k starts at k s and is
// min(6000, L - k s) long; the first is always a candidate, every other one only if it has >= 2500 nt, so
// n_cand = 1 + max(0, (L - 2500) / s).  At s = 6000 this is seq_windows(6000, 2500) (sequence.py:150-167):
// L / 6000 + (L % 6000 >= 2500), at least 1.  s = 0 stands for --single-window: the first window only.
__device__ __forceinline__ int64_t candidate_windows(int64_t L, int64_t step) {
  if (step == 0) return 1;
  return 1 + (L > kMinTail ? (L - kMinTail) / step : 0);
}

// Windows start every `window_step` bytes of the stripped contig (6000: the reference's windows; smaller: overlapping windows of
// a score profile, each candidate's N count re-reads its 6000 bytes, i.e. ~6000 / step reads per byte; 0: --single-window).
// kWrite = false: counts[c] = kept windows of contig c (-1 if its byte range is reversed).
// kWrite = true : offsets = the scanned counts; contig c writes its kept windows to win_start / win_len [offsets[c], offsets[c+1]).
// kReverse: the windows of the contig's reverse complement rc(S) (genomad/sequence.py:41-43).  Candidate k is laid from the
// stripped end: it is rc(S)[k step, k step + len_k), i.e. the forward segment [L - k step - len_k, L - k step), and
// win_start / win_len name that segment.  rc maps 'N' to 'N', so the N rule counts the segment's 'N' bytes.
template <bool kWrite, bool kReverse>
__device__ __forceinline__ void contig_plan(const uint8_t* __restrict__ seq, const int64_t* __restrict__ seq_offsets,
                                            int window_step, int32_t* __restrict__ offsets, int64_t* __restrict__ win_start,
                                            int32_t* __restrict__ win_len) {
  __shared__ unsigned long long s_best;
  __shared__ int s_keep[kPlanWarps];
  const int c = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t s0 = seq_offsets[c], s1 = seq_offsets[c + 1];
  int64_t base = 0, n_kept = 0;
  if (kWrite) {
    base = offsets[c];
    n_kept = offsets[c + 1] - base;
    if (n_kept == 0) return;                           // empty after stripping: nothing to re-read
  } else if (s1 < s0) {
    if (threadIdx.x == 0) offsets[c] = -1;
    return;
  }
  const int64_t first = block_find_non_n<false>(seq, s0, s1, &s_best);
  if (first < 0) {                                     // empty or nothing but n/N (only reached by the count pass)
    if (!kWrite && threadIdx.x == 0) offsets[c] = 0;
    return;
  }
  const int64_t L = block_find_non_n<true>(seq, first, s1, &s_best) + 1 - first;
  const int64_t step = window_step;
  const int64_t n_cand = candidate_windows(L, step);
  auto wlen = [&](int64_t w) { return static_cast<int32_t>(min(static_cast<int64_t>(kWindow), L - w * step)); };
  auto wbeg = [&](int64_t w) { return kReverse ? first + L - w * step - wlen(w) : first + w * step; };
  if (kWrite && n_kept == n_cand) {                    // nothing dropped by the N rule: window k is candidate k
    for (int64_t w = threadIdx.x; w < n_cand; w += blockDim.x) {
      win_start[base + w] = wbeg(w);
      win_len[base + w] = wlen(w);
    }
    return;
  }
  if (kWrite && threadIdx.x == 0) { win_start[base] = wbeg(0); win_len[base] = wlen(0); }     // the first window is exempt
  int64_t kept = 1;                                    // windows kept so far, identical in every thread
  for (int64_t w0 = 1; w0 < n_cand; w0 += kPlanWarps) {   // rounds of one candidate per warp, in order
    const int64_t w = w0 + warp;
    int keep = 0;
    if (w < n_cand) {
      const int64_t a = wbeg(w);
      keep = warp_count_N(seq, a, a + wlen(w)) <= kMaxN;
    }
    if (lane == 0) s_keep[warp] = keep;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int i = 0; i < kPlanWarps; ++i) { before += i < warp ? s_keep[i] : 0; total += s_keep[i]; }
    if (kWrite && keep && lane == 0) {
      win_start[base + kept + before] = wbeg(w);
      win_len[base + kept + before] = wlen(w);
    }
    kept += total;
    __syncthreads();                                   // s_keep is rewritten by the next round
  }
  if (!kWrite && threadIdx.x == 0) offsets[c] = kept > INT32_MAX ? kCountOverflow : static_cast<int32_t>(kept);
}

template <bool kWrite>
__global__ void __launch_bounds__(kPlanThreads)
contig_plan_kernel(const uint8_t* __restrict__ seq, const int64_t* __restrict__ seq_offsets, int window_step,
                   int32_t* __restrict__ offsets, int64_t* __restrict__ win_start, int32_t* __restrict__ win_len) {
  contig_plan<kWrite, false>(seq, seq_offsets, window_step, offsets, win_start, win_len);
}
template <bool kWrite>
__global__ void __launch_bounds__(kPlanThreads)
contig_plan_rc_kernel(const uint8_t* __restrict__ seq, const int64_t* __restrict__ seq_offsets, int window_step,
                      int32_t* __restrict__ offsets, int64_t* __restrict__ win_start, int32_t* __restrict__ win_len) {
  contig_plan<kWrite, true>(seq, seq_offsets, window_step, offsets, win_start, win_len);
}

// offsets[0, n) = per-contig window counts -> exclusive prefix sums in place, offsets[n] = the total, or kPlanOverflow if it
// (or one contig's count, kCountOverflow) exceeds INT32_MAX, or kPlanBadOffsets if a count is otherwise negative.  One CTA
// walks the array in rounds of kScanThreads * kScanPer counts with a 64-bit carry.
__global__ void __launch_bounds__(kScanThreads) contig_scan_kernel(int32_t* __restrict__ offsets, int n) {
  __shared__ long long s_warp[kScanThreads / 32];
  __shared__ long long s_carry;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  long long carry = 0;
  int bad = 0, over = 0;
  for (long long r0 = 0; r0 < n; r0 += static_cast<long long>(kScanThreads) * kScanPer) {
    const long long i0 = r0 + static_cast<long long>(threadIdx.x) * kScanPer;
    int v[kScanPer];
    long long t = 0;
#pragma unroll
    for (int k = 0; k < kScanPer; ++k) {
      v[k] = i0 + k < n ? offsets[i0 + k] : 0;
      if (v[k] == kCountOverflow) { over = 1; v[k] = 0; }
      else if (v[k] < 0) { bad = 1; v[k] = 0; }
      t += v[k];
    }
    long long incl = t;                                // inclusive scan of the per-thread sums within the warp
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      long long x = s_warp[lane], s = x;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, s, d);
        if (lane >= d) s += y;
      }
      s_warp[lane] = s - x;                            // exclusive prefix of the warp totals
    }
    __syncthreads();
    long long run = carry + s_warp[warp] + incl - t;
#pragma unroll
    for (int k = 0; k < kScanPer; ++k) {
      if (i0 + k < n) offsets[i0 + k] = static_cast<int32_t>(run);
      run += v[k];
    }
    if (threadIdx.x == kScanThreads - 1) s_carry = run;   // the last thread ends the round
    __syncthreads();                                   // also: every thread has read s_warp before the next round rewrites it
    carry = s_carry;
  }
  bad = __syncthreads_or(bad);
  over = __syncthreads_or(over);
  if (threadIdx.x == 0)
    offsets[n] = bad ? kPlanBadOffsets : over || carry > 0x7fffffffLL ? kPlanOverflow : static_cast<int32_t>(carry);
}

// One CTA per window: stage the window's bytes (any start address) in shared memory with aligned 16-byte loads, then write
// the 6000-byte row with 16-byte stores: ASCII upper-case of 'a'..'z' only, 'N' past the window's length.  Lengths outside
// [0, 6000] are clamped to it.
__global__ void __launch_bounds__(kGatherThreads)
gather_windows_kernel(const uint8_t* __restrict__ seq, const int64_t* __restrict__ win_start, const int32_t* __restrict__ win_len,
                      uint8_t* __restrict__ out) {
  __shared__ __align__(16) uint32_t s_w[(kWindow + 32) / 4];
  const int64_t w = blockIdx.x;
  const int len = min(max(win_len[w], 0), kWindow);
  const uint8_t* src = seq + win_start[w];
  const int shift = static_cast<int>(reinterpret_cast<uintptr_t>(src) & 15);
  const uint4* v0 = reinterpret_cast<const uint4*>(src - shift);
  const int nvec = len > 0 ? (shift + len + 15) / 16 : 0;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) reinterpret_cast<uint4*>(s_w)[i] = v0[i];
  __syncthreads();
  const int q0 = shift >> 2, r8 = 8 * (shift & 3);
  uint8_t* dst = out + w * kWindow;
  for (int i = threadIdx.x; i < kWindow / 16; i += blockDim.x) {
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = 16 * i + 4 * k;                    // first byte of this word in the window
      const int q = q0 + j / 4;
      uint32_t x = __funnelshift_r(s_w[q], s_w[q + 1], r8);      // bytes j .. j+3 (past len: stale, replaced below)
      const int e = len - j;
      const uint32_t in = e >= 4 ? 0xffffffffu : e <= 0 ? 0u : 0xffffffffu >> (32 - 8 * e);
      x = (x & in) | (0x4e4e4e4eu & ~in);
      const uint32_t lower = __vcmpgeu4(x, 0x61616161u) & __vcmpleu4(x, 0x7a7a7a7au);
      o[k] = x - (lower & 0x20202020u);
    }
    *reinterpret_cast<uint4*>(dst + 16 * i) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// upper(comp(c)) in each byte: comp is Sequence.rc()'s table (ACTGNactgn -> TGACNtgacn, every other byte unchanged), and upper()
// changes 'a'..'z' only.  Upper-casing first leaves A, C, G, T exactly where comp acts ('N' and 'n' become 'N' either way);
// then A <-> T is ^ 0x15 and C <-> G is ^ 0x04.
__device__ __forceinline__ uint32_t rc_upper4(uint32_t x) {
  const uint32_t lower = __vcmpgeu4(x, 0x61616161u) & __vcmpleu4(x, 0x7a7a7a7au);
  const uint32_t u = x - (lower & 0x20202020u);
  const uint32_t at = __vcmpeq4(u, 0x41414141u) | __vcmpeq4(u, 0x54545454u);
  const uint32_t cg = __vcmpeq4(u, 0x43434343u) | __vcmpeq4(u, 0x47474747u);
  return u ^ (at & 0x15151515u) ^ (cg & 0x04040404u);
}

// gather_windows_kernel for the windows of the reverse complement: (start, length) names the window's forward segment seg, and
// row byte j = upper(comp(seg[len - 1 - j])), 'N' past len.  The staged copy starts 16 bytes into s_w so that a word read
// backwards from the segment's first byte stays inside the buffer; each output word is the staged word that ends at
// seg[len - 1 - j], byte-reversed.
__global__ void __launch_bounds__(kGatherThreads)
gather_windows_rc_kernel(const uint8_t* __restrict__ seq, const int64_t* __restrict__ win_start,
                         const int32_t* __restrict__ win_len, uint8_t* __restrict__ out) {
  __shared__ __align__(16) uint32_t s_w[(kWindow + 48) / 4];
  const int64_t w = blockIdx.x;
  const int len = min(max(win_len[w], 0), kWindow);
  const uint8_t* src = seq + win_start[w];
  const int shift = static_cast<int>(reinterpret_cast<uintptr_t>(src) & 15);
  const uint4* v0 = reinterpret_cast<const uint4*>(src - shift);
  const int nvec = len > 0 ? (shift + len + 15) / 16 : 0;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) reinterpret_cast<uint4*>(s_w)[i + 1] = v0[i];
  __syncthreads();
  uint8_t* dst = out + w * kWindow;
  const int last = 16 + shift + len - 4;               // staged byte index of seg[len - 4]
  for (int i = threadIdx.x; i < kWindow / 16; i += blockDim.x) {
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = 16 * i + 4 * k;                    // first byte of this word in the row
      const int e = len - j;
      uint32_t x = 0x4e4e4e4eu;
      if (e > 0) {
        const int p = last - j;                        // >= 13: staged bytes p .. p+3 = seg[len-4-j .. len-1-j]
        x = __byte_perm(__funnelshift_r(s_w[p >> 2], s_w[(p >> 2) + 1], 8 * (p & 3)), 0, 0x0123);
        const uint32_t in = e >= 4 ? 0xffffffffu : 0xffffffffu >> (32 - 8 * e);   // bytes before seg's start: 'N'
        x = rc_upper4((x & in) | (0x4e4e4e4eu & ~in));
      }
      o[k] = x;
    }
    *reinterpret_cast<uint4*>(dst + 16 * i) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace gnm
