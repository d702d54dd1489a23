// K0: ASCII -> 4-mer tokens, and K0+K1 fused: ASCII/tokens -> first conv layer output.
//
// Reference semantics:
//   tokenize_dna            genomad/sequence.py:170-193  (closed form: tok = 0 if any of the 4 bytes
//                           is not one of 'A','C','G','T' (65,67,71,84), else 1 + base-4 value)
//   one-hot + Conv1D#1      genomad/neural_network/model.py:11, igloo.py:45-48
//                           y1[t] = lrelu(b + sum_{j=0..5, t-5+j>=0} W1[j][tok[t-5+j]][:])
//                           (causal zero padding adds nothing -- it is NOT token 0)
#pragma once
#include "common.cuh"

namespace gnm {

// 2-bit code of an upper-case nucleotide byte, or 4 for anything else
__device__ __forceinline__ uint32_t base_code(uint8_t b) {
  return b == 'A' ? 0u : b == 'C' ? 1u : b == 'G' ? 2u : b == 'T' ? 3u : 4u;
}
__device__ __forceinline__ uint16_t kmer_token(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
  const uint32_t bad = (c0 | c1 | c2 | c3) & 4u;
  const uint32_t v = 1u + 64u * c0 + 16u * c1 + 4u * c2 + c3;
  return bad ? uint16_t(0) : uint16_t(v);
}

// A caller's token as a table row index: tf.one_hot(x, 257) turns a token above 256 into an all-zero row, so such a token
// contributes nothing, exactly like the causal padding (-1).
__device__ __forceinline__ int vocab_token(uint32_t v) { return v < kVocab ? static_cast<int>(v) : -1; }

// Layer 1's triple-table shortcut for caller-supplied tokens: the row ((tk0-1) << 4) | ((tk2-1) & 15) holds
// W1[j][k0] + W1[j+1][k1] + W1[j+2][k2] for the three overlapping 4-mers of one all-ACGT 6-base word, so it may replace the
// three rows only when tk0, tk1, tk2 are such 4-mers (tokenizer output always is; arbitrary tokens mostly are not).
// 0xFFFF = take the three-row fallback.
__device__ __forceinline__ int triple_code_checked(int tk0, int tk1, int tk2) {
  const bool word = tk0 > 0 && tk1 > 0 && tk2 > 0 && ((tk0 - 1) & 15) == ((tk2 - 1) >> 4) &&
                    tk1 - 1 == ((((tk0 - 1) & 63) << 2) | (((tk2 - 1) >> 2) & 3));
  return word ? (((tk0 - 1) << 4) | ((tk2 - 1) & 15)) : 0xFFFF;
}

// ------------------------------------------------------------------------------------------
// K0 (stand-alone): one CTA per (window, 2048-token segment).  Bytes are staged through shared
// memory with 16-byte coalesced loads; every thread then emits 8 consecutive tokens as one
// 16-byte store.  Pure byte/integer work, HBM-bound: 6000 B in + 11994 B out per window.
// ------------------------------------------------------------------------------------------
constexpr int kEncSeg = 2048;                         // tokens per CTA
constexpr int kEncThreads = kEncSeg / 8;              // 256

__global__ void __launch_bounds__(kEncThreads)
encode_tokens_kernel(const uint8_t* __restrict__ ascii, uint16_t* __restrict__ tokens, int n_windows) {
  __shared__ __align__(16) uint8_t s_b[kEncSeg + 16];
  const int w = blockIdx.y;
  const int t0 = blockIdx.x * kEncSeg;
  const uint8_t* src = ascii + static_cast<size_t>(w) * kWindow;
  // window rows are 6000 B apart: 16-byte aligned (6000 = 375 * 16) as long as the base is.
  for (int i = threadIdx.x; i < (kEncSeg + 16) / 16; i += blockDim.x) {
    const int off = t0 + i * 16;
    uint4 v = make_uint4(0x4E4E4E4Eu, 0x4E4E4E4Eu, 0x4E4E4E4Eu, 0x4E4E4E4Eu);   // 'N'
    if (off + 16 <= kWindow) {
      v = *reinterpret_cast<const uint4*>(src + off);
    } else if (off < kWindow) {
      uint8_t tmp[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) tmp[k] = (off + k < kWindow) ? src[off + k] : uint8_t('N');
      v = *reinterpret_cast<uint4*>(tmp);
    }
    *reinterpret_cast<uint4*>(s_b + i * 16) = v;
  }
  __syncthreads();
  const int lt = threadIdx.x * 8;            // first token (within the segment) of this thread
  uint32_t c[11];
#pragma unroll
  for (int k = 0; k < 11; ++k) c[k] = base_code(s_b[lt + k]);
  uint16_t out[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) out[k] = kmer_token(c[k], c[k + 1], c[k + 2], c[k + 3]);
  uint16_t* dst = tokens + static_cast<size_t>(w) * kTok;
  const int t = t0 + lt;
  // token rows are 5997*2 B apart -> not 16-byte aligned in general: scalar stores
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if (t + k < kTok) dst[t + k] = out[k];
}

// ------------------------------------------------------------------------------------------
// K0+K1 fused: one CTA per (window, 256-position segment).  Tokens are computed into shared
// memory (from ASCII, or copied from a token buffer), then one warp per position produces the
// 128-channel activation row and writes its four planes (768 B, layout in common.cuh).
//
//   y1[t] = lrelu( (A + B) + bias ),   A = (W1[0][k0] + W1[1][k1]) + W1[2][k2],  B = (W1[3][k3] + W1[4][k4]) + W1[5][k5]
//
// with k_j = tok[t-5+j] and padded taps contributing exactly 0.  Tokens t-5, t-4, t-3 are the 4-mers
// of 6 consecutive bases, so A has only 4^6 = 4096 possible values when those bases are all ACGT, and
// likewise B: two 2 MB "triple" tables (built on the host with the same fp32 operation order, so a
// table hit is bit-identical to the three-row sum) replace six 512-byte row reads by two.  Positions
// next to the window start, or touching a non-ACGT base, fall back to the single-row table.  Tokens
// supplied by the caller (kFromAscii = false) may be anything: values above 256 become padding (the
// zero row of tf.one_hot), and a half takes its triple row only when its three tokens are the 4-mers of
// one 6-base word.
// ------------------------------------------------------------------------------------------
constexpr int kEmbSeg = 256;
constexpr int kEmbThreads = 256;
constexpr int kTriple = 4096;
static_assert(kEmbThreads == kEmbSeg, "embed_conv1_kernel computes one position's table codes per thread");

// Integrated gradients (attr.cuh, DESIGN.md "Integrated gradients") run layer 1 at inputs on the straight line from a
// baseline x' to the window x.  Conv1D #1 is linear in its one-hot input, so the pre-activation there is
//   alpha * S_tok + (1 - alpha) * S_base + b,   S_tok = the (A + B) sum below,
//   S_base = 0 (kIgZero: all-zero one-hot rows) or sum_{j: t-5+j >= 0} W1[j][0] (kIgN: the all-N window, token 0 everywhere;
//            summed in the fallback's order, so it is bitwise the all-N window's A + B).
// computed as fmaf(alpha, S_tok, fmaf(1 - alpha, S_base, b)) (kIgN) or fmaf(alpha, S_tok, b) (kIgZero): at alpha = 1 that is
// exactly the (A + B) + b of the plain kernel, so the row is bitwise the plain kernel's.
constexpr int kIgZero = 0, kIgN = 1;

// Row `row` of an interpolated launch: window row / m at alpha_k = (k + 1/2) / m, k = row mod m (midpoint rule); m = 0 is the
// baseline itself (alpha = 0).
struct IgRow {
  int win; float alpha, beta;                // beta = 1 - alpha, both rounded once from exact numerators
};
__device__ __forceinline__ IgRow ig_row(int row, int m) {
  if (m <= 0) return {0, 0.f, 1.f};
  const int k = row % m;
  return {row / m, (static_cast<float>(k) + 0.5f) / static_cast<float>(m), (static_cast<float>(m - k) - 0.5f) / static_cast<float>(m)};
}

// The body of embed_conv1_kernel; kIg (ASCII input only) adds the interpolation of the pre-activation.  win: the window whose
// bytes / tokens are read, out_row: the output row.
template <bool kFromAscii, bool kIg>
__device__ __forceinline__ void embed_conv1_body(const uint8_t* __restrict__ ascii, const uint16_t* __restrict__ tokens_in,
                                                 const float* __restrict__ table, const float* __restrict__ triple,
                                                 const float* __restrict__ bias, uint8_t* __restrict__ y_out, int win, int out_row,
                                                 float alpha, float beta, int baseline, DeviceStatus* status) {
  __shared__ int16_t s_tok[kEmbSeg + 8];    // s_tok[i] = token at position t0 - 5 + i, or -1 (causal pad)
  __shared__ uint8_t s_b[kEmbSeg + 16];
  __shared__ int s_code[kEmbSeg];           // per position: (A code | B code << 16), 0xFFFF in a half = that half needs the 3-row fallback
  const int w = win;
  const int t0 = blockIdx.x * kEmbSeg;
  if (kFromAscii) {
    const uint8_t* src = ascii + static_cast<size_t>(w) * kWindow;
    for (int i = threadIdx.x; i < kEmbSeg + 8 + 3; i += blockDim.x) {
      const int p = t0 - 5 + i;
      s_b[i] = (p >= 0 && p < kWindow) ? src[p] : uint8_t('N');
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kEmbSeg + 5; i += blockDim.x) {
      const int p = t0 - 5 + i;
      int16_t tk = -1;
      if (p >= 0 && p < kTok)
        tk = static_cast<int16_t>(kmer_token(base_code(s_b[i]), base_code(s_b[i + 1]),
                                             base_code(s_b[i + 2]), base_code(s_b[i + 3])));
      s_tok[i] = tk;
    }
  } else {
    const uint16_t* src = tokens_in + static_cast<size_t>(w) * kTok;
    for (int i = threadIdx.x; i < kEmbSeg + 5; i += blockDim.x) {
      const int p = t0 - 5 + i;
      s_tok[i] = static_cast<int16_t>((p >= 0 && p < kTok) ? vocab_token(src[p]) : -1);
    }
  }
  __syncthreads();
  // Triple-table codes once per position (one thread each) instead of once per lane of the warp that produces the row: the
  // row loop below was issue-bound (83 % of the issue slots, ~115 warp instructions per position, a third of them this
  // token logic executed redundantly by all 32 lanes).
  {
    const int i = threadIdx.x;                         // kEmbThreads == kEmbSeg
    int ca, cb;
    if (kFromAscii) {                                  // tokens made from bytes here are consistent 4-mers by construction
      const int tk0 = s_tok[i], tk2 = s_tok[i + 2], tk3 = s_tok[i + 3], tk5 = s_tok[i + 5];
      ca = (tk0 > 0 && tk2 > 0) ? (((tk0 - 1) << 4) | ((tk2 - 1) & 15)) : 0xFFFF;    // bases t-5 .. t all ACGT (implies tk1 > 0)
      cb = (tk3 > 0 && tk5 > 0) ? (((tk3 - 1) << 4) | ((tk5 - 1) & 15)) : 0xFFFF;    // bases t-2 .. t+3 all ACGT (implies tk4 > 0)
    } else {
      ca = triple_code_checked(s_tok[i], s_tok[i + 1], s_tok[i + 2]);
      cb = triple_code_checked(s_tok[i + 3], s_tok[i + 4], s_tok[i + 5]);
    }
    s_code[i] = ca | (cb << 16);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float4 b4 = reinterpret_cast<const float4*>(bias)[lane];
  const float4* tab4 = reinterpret_cast<const float4*>(table);
  const float4* tri4 = reinterpret_cast<const float4*>(triple);
  auto row = [&](int j, int tk) -> float4 {
    return tk >= 0 ? __ldg(tab4 + (static_cast<size_t>(j) * kVocab + tk) * (kC / 4) + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  auto add4 = [](float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); };
  float amax = 0.f;
  const int i_end = min(kEmbSeg, kTok - t0);
  for (int i = warp; i < i_end; i += kEmbThreads / 32) {
    const int t = t0 + i;
    const int code = s_code[i];
    const int ca = code & 0xFFFF, cb = static_cast<unsigned>(code) >> 16;
    float4 A, B;
    if (ca != 0xFFFF) A = __ldg(tri4 + static_cast<size_t>(ca) * (kC / 4) + lane);
    else A = add4(add4(row(0, s_tok[i]), row(1, s_tok[i + 1])), row(2, s_tok[i + 2]));
    if (cb != 0xFFFF) B = __ldg(tri4 + (static_cast<size_t>(kTriple) + cb) * (kC / 4) + lane);
    else B = add4(add4(row(3, s_tok[i + 3]), row(4, s_tok[i + 4])), row(5, s_tok[i + 5]));
    float4 a = add4(A, B);
    if (kIg) {
      float4 b = b4;
      if (baseline == kIgN) {                          // S_base: token 0 at every tap inside the window, in the fallback's order
        const auto r0 = [&](int j) { return row(j, t - 5 + j >= 0 ? 0 : -1); };
        const float4 sb = add4(add4(add4(r0(0), r0(1)), r0(2)), add4(add4(r0(3), r0(4)), r0(5)));
        b = make_float4(fmaf(beta, sb.x, b4.x), fmaf(beta, sb.y, b4.y), fmaf(beta, sb.z, b4.z), fmaf(beta, sb.w, b4.w));
      }
      a = make_float4(fmaf(alpha, a.x, b.x), fmaf(alpha, a.y, b.y), fmaf(alpha, a.z, b.z), fmaf(alpha, a.w, b.w));
      a.x = kActScale * lrelu(a.x); a.y = kActScale * lrelu(a.y);
      a.z = kActScale * lrelu(a.z); a.w = kActScale * lrelu(a.w);
    } else {
    // Y = 32 * y1; planes: hi16, lo16 (w_v, gather), lo8 / hi8 (conv2 correction passes)
    a.x = kActScale * lrelu(a.x + b4.x); a.y = kActScale * lrelu(a.y + b4.y);
    a.z = kActScale * lrelu(a.z + b4.z); a.w = kActScale * lrelu(a.w + b4.w);
    }
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))));
    __half2 h01, h23, l01, l23;
    split2_f16(a.x, a.y, h01, l01);
    split2_f16(a.z, a.w, h23, l23);
    const float2 fa = __half22float2(h01), fb = __half22float2(h23);
    const float f0 = fa.x, f1 = fa.y, f2 = fb.x, f3 = fb.y;
    uint8_t* rowp = y_out + (static_cast<size_t>(out_row) * kTok + t) * kRowBytes;
    *reinterpret_cast<uint2*>(rowp + kOffHi16 + lane * 8) =
        make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
    *reinterpret_cast<uint2*>(rowp + kOffLo16 + lane * 8) =
        make_uint2(*reinterpret_cast<const uint32_t*>(&l01), *reinterpret_cast<const uint32_t*>(&l23));
    // e4m3 pairs (lo8[c], hi8[c]) of this lane's 4 channels: 8 contiguous bytes
    *reinterpret_cast<uint2*>(rowp + kOffP8 + lane * 8) = make_uint2(
        static_cast<uint32_t>(pack_e4m3x2((a.x - f0) * kLo8Scale, f0 * kHi8Scale)) |
            (static_cast<uint32_t>(pack_e4m3x2((a.y - f1) * kLo8Scale, f1 * kHi8Scale)) << 16),
        static_cast<uint32_t>(pack_e4m3x2((a.z - f2) * kLo8Scale, f2 * kHi8Scale)) |
            (static_cast<uint32_t>(pack_e4m3x2((a.w - f3) * kLo8Scale, f3 * kHi8Scale)) << 16));
  }
  flag_act_overflow(status, amax, kHi8Limit, 1);
}

template <bool kFromAscii>
__global__ void __launch_bounds__(kEmbThreads)
embed_conv1_kernel(const uint8_t* __restrict__ ascii, const uint16_t* __restrict__ tokens_in,
                   const float* __restrict__ table,   // [6][257][128]
                   const float* __restrict__ triple,  // [2][4096][128]: A-table, B-table
                   const float* __restrict__ bias,    // [128]
                   uint8_t* __restrict__ y_out,       // [n][5997][768 B] activation rows (hi16 | lo16 | e4m3 pairs)
                   int n_windows, DeviceStatus* status) {
  embed_conv1_body<kFromAscii, false>(ascii, tokens_in, table, triple, bias, y_out, blockIdx.y, blockIdx.y, 1.f, 0.f, 0, status);
}

// Interpolated layer 1 (integrated gradients): grid (24, rows); row r is window r / m of `ascii` at alpha_k (ig_row), so a
// chunk holds each window's bytes once, not m copies.  m = 0: every row is the baseline x' (alpha = 0).
__global__ void __launch_bounds__(kEmbThreads)
embed_conv1_ig_kernel(const uint8_t* __restrict__ ascii, const float* __restrict__ table, const float* __restrict__ triple,
                      const float* __restrict__ bias, uint8_t* __restrict__ y_out, int m, int baseline, DeviceStatus* status) {
  const IgRow r = ig_row(blockIdx.y, m);
  embed_conv1_body<true, true>(ascii, nullptr, table, triple, bias, y_out, r.win, blockIdx.y, r.alpha, r.beta, baseline, status);
}

}  // namespace gnm
