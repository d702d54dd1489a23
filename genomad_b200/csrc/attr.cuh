// Attribution pass: attr[t] = d log p_c / d x[t, tok[t]] for the one-hot input x of the first Conv1D (gradient x input), the
// exact backward of the forward as written.  The tensor-core parts are instantiations of conv_t.cuh's body (kConvRoute: the
// w_v pass storing where each pooled maximum sits; kConvBwd: the conv pass over time-reversed gradient rows against W[j]^T);
// everything here runs on the CUDA cores in fp32 with a fixed summation order and no atomics, so a window's attributions do not
// depend on its batch, its chunk or the GPU count.
//
// Backward, per window (DESIGN.md, "Attributions"):
//   head     g_logits = e_c - p, as -p_i and, for the target, the sum of the other p_i (never 1 - p_c, which cancels
//            when p_c is near 1); back through Dense(C), BN1 + ReLU, Dense(512), BN0 + ReLU, Dense(512)  -> g_out0, g_out1
//            (C = 3 and the shipped tail, or a trained head's last three layers)
//   IGLOO k  out = alpha^T q, alpha = softmax(mpi w_qk), q = maxpool8(y w_v)
//            g_q[p,c] = alpha[p] g_out[c];  g_alpha[p] = sum_c g_out[c] q[p,c];  g_logit = alpha (g_alpha - <alpha, g_alpha>)
//            g_mpi = w_qk g_logit (sgemm_epi_kernel);  g_y[t] = sum over the (p,c) routed to t of g_q[p,c] w_v[:,c]
//                                                            + sum over the patch entries (i,k) on t of g_mpi[i] Wf[i,k,:]
//   convs    g_z = g_y * lrelu'(y);  g_yprev[s] = sum_j g_z[s+5-j] W[j]^T  (conv_t_attr_kernel<kConvBwd>, rows reversed)
//   layer 1  attr[t] = sum_{u=t}^{min(t+5,5996)} <g_z1[u], W1[t-u+5, tok[t], :]>
// From g_z3 on, the gradient is carried times a per-window power of two s_w (max |g_z3| s_w in [0.25, 0.5)) so that the conv
// operand formats (common.cuh) see values in their range; layer 1 divides it out.  conv3's backward output gets a power of two
// of its own, s2 (max |s_w g_z2| s2 in [1, 2)), for the operand rows conv2's backward pass reads; that pass divides it out.
#pragma once
#include "common.cuh"
#include "conv_t.cuh"
#include "encode.cuh"
#include "head.cuh"
#include "igloo.cuh"

namespace gnm {

constexpr int kAttrPosBlock = 64;                                         // positions per CTA of the IGLOO backward kernel
constexpr int kAttrPosBlocks = (kTok + kAttrPosBlock - 1) / kAttrPosBlock; // 94
constexpr int kAttrSeg = 256;                                             // positions per CTA of the pack / layer-1 kernels

// warp sum in a fixed butterfly order (every lane gets the same bits)
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// ------------------------------------------------------------------------------------------------ head
// The class arguments of the head-gradient and log p kernels, target c and class count C, travel in one int, tc = c | C << 8:
// the kernels keep the parameter lists (and symbols) they had when C was always 3.
__host__ __device__ constexpr int attr_classes(int target, int C) { return target | (C << 8); }
__device__ __forceinline__ int attr_target_of(int tc) { return tc & 0xff; }
__device__ __forceinline__ int attr_count_of(int tc) { return tc >> 8; }

// One window per CTA, 256 threads.  g_out[w][0..255] = d log p_c / d h0 (h0 = [out0 | out1]), unscaled, through a C-class head
// (2 <= C <= 32): the shipped tail at C = 3 (d2w, d1w, bn1_scale, h2 the handle's) or a trained head (gnm_head's d2w, d1w and
// folded BN scale, h2 its hidden rows).  Dense(512) #0 and its BN are the encoder's in both cases.
__global__ void __launch_bounds__(256)
attr_head_backward_kernel(const float* __restrict__ probs,      // [n][C]
                          const float* __restrict__ h1, const float* __restrict__ h2,   // [n][512] (post-ReLU)
                          const float* __restrict__ d2w,        // [512][C]
                          const float* __restrict__ d1w,        // [512][512]
                          const float* __restrict__ bn1_scale,  // [512]
                          const float* __restrict__ d0w,        // [256][512]
                          const float* __restrict__ bn0_scale,  // [512]
                          int tc,                               // attr_classes(target, C)
                          float* __restrict__ g_out) {
  __shared__ float s_a1[kHidden], s_a0[kHidden], s_gl[kHeadMaxClasses];
  const int w = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int target = attr_target_of(tc), C = attr_count_of(tc);
  // g_logits = e_c - p with the target's component as the sum of the other probabilities (ascending i), not 1 - p_c:
  // values just below 1 are 2^-24 apart, so 1 - p_c cancels for a window classified confidently as the target and is
  // exactly 0 once p_c rounds to 1.0f (log-odds margin ~17.3), while the off-target p_i keep their relative precision
  if (tid == 0) {
    float other = 0.f;
    for (int i = 0; i < C; ++i) {
      const float p = probs[static_cast<size_t>(w) * C + i];
      s_gl[i] = -p;
      if (i != target) other += p;
    }
    s_gl[target] = other;
  }
  __syncthreads();
  for (int k = tid; k < kHidden; k += 256) {                    // gl[0] w[k][0], then one fmaf per class, ascending
    const float* wk = d2w + static_cast<size_t>(k) * C;
    float g = s_gl[0] * wk[0];
    for (int i = 1; i < C; ++i) g = fmaf(s_gl[i], wk[i], g);
    s_a1[k] = h2[static_cast<size_t>(w) * kHidden + k] > 0.f ? g * bn1_scale[k] : 0.f;
  }
  __syncthreads();
  for (int j = warp; j < kHidden; j += 8) {                     // g_h1[j] = sum_k d1w[j][k] g_a1[k]
    const float* row = d1w + static_cast<size_t>(j) * kHidden;
    float a = 0.f;
#pragma unroll 4
    for (int k = lane; k < kHidden; k += 32) a = fmaf(row[k], s_a1[k], a);
    a = warp_sum(a);
    if (lane == 0) s_a0[j] = h1[static_cast<size_t>(w) * kHidden + j] > 0.f ? a * bn0_scale[j] : 0.f;
  }
  __syncthreads();
  for (int m = warp; m < 256; m += 8) {                         // g_h0[m] = sum_j d0w[m][j] g_a0[j]
    const float* row = d0w + static_cast<size_t>(m) * kHidden;
    float a = 0.f;
#pragma unroll 4
    for (int j = lane; j < kHidden; j += 32) a = fmaf(row[j], s_a0[j], a);
    a = warp_sum(a);
    if (lane == 0) g_out[static_cast<size_t>(w) * 256 + m] = a;
  }
}

// One window per CTA, 256 threads.  g_out[w][0..255] = d D_c / d h0 from g_h1 = d D_c / d h1 (nv_grad_kernel's fp32 rows): the
// last stage of attr_head_backward_kernel, in its order.
__global__ void __launch_bounds__(256)
attr_novelty_backward_kernel(const float* __restrict__ g_h1,      // [n][512]
                             const float* __restrict__ h1,        // [n][512] (post-ReLU)
                             const float* __restrict__ d0w,       // [256][512]
                             const float* __restrict__ bn0_scale, // [512]
                             float* __restrict__ g_out) {
  __shared__ float s_a0[kHidden];
  const int w = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int j = tid; j < kHidden; j += 256) {
    const size_t o = static_cast<size_t>(w) * kHidden + j;
    s_a0[j] = h1[o] > 0.f ? g_h1[o] * bn0_scale[j] : 0.f;
  }
  __syncthreads();
  for (int m = warp; m < 256; m += 8) {                         // g_h0[m] = sum_j d0w[m][j] g_a0[j]
    const float* row = d0w + static_cast<size_t>(m) * kHidden;
    float a = 0.f;
#pragma unroll 4
    for (int j = lane; j < kHidden; j += 32) a = fmaf(row[j], s_a0[j], a);
    a = warp_sum(a);
    if (lane == 0) g_out[static_cast<size_t>(w) * 256 + m] = a;
  }
}

// ------------------------------------------------------------------------------------------------ IGLOO: attention part
// One window per CTA, 256 threads: alpha = softmax(logits) (as attention_kernel), g_alpha, g_logit -> [n][752] rows.
__global__ void __launch_bounds__(256)
attr_igloo_prep_kernel(const float* __restrict__ logits,    // [n][752]
                       const float* __restrict__ q,         // [n][749][128]
                       const float* __restrict__ g_out,     // [n][256] + column offset of this IGLOO kernel
                       float* __restrict__ alpha_out,       // [n][752]
                       float* __restrict__ g_logit) {       // [n][752]
  __shared__ __align__(16) float s_go[kC];                        // read as float4
  __shared__ float s_al[kPooled], s_ga[kPooled], s_red[8];
  const int w = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* lrow = logits + static_cast<size_t>(w) * kLogitsLd;
  if (tid < kC) s_go[tid] = g_out[static_cast<size_t>(w) * 256 + tid];
  float m = -INFINITY;
  for (int g = tid; g < kPooled; g += 256) { const float v = lrow[g]; s_al[g] = v; m = fmaxf(m, v); }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if (lane == 0) s_red[warp] = m;
  __syncthreads();
  m = s_red[0];
  for (int i = 1; i < 8; ++i) m = fmaxf(m, s_red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int g = tid; g < kPooled; g += 256) { const float e = expf(s_al[g] - m); s_al[g] = e; sum += e; }
  sum = warp_sum(sum);
  if (lane == 0) s_red[warp] = sum;
  __syncthreads();
  sum = ((s_red[0] + s_red[1]) + (s_red[2] + s_red[3])) + ((s_red[4] + s_red[5]) + (s_red[6] + s_red[7]));
  const float inv = 1.f / sum;
  __syncthreads();
  for (int g = tid; g < kPooled; g += 256) s_al[g] *= inv;
  // g_alpha[p] = sum_c g_out[c] q[p,c]: one warp per pooled row, lanes over channels
  const float4 go = reinterpret_cast<const float4*>(s_go)[lane];
  for (int g = warp; g < kPooled; g += 8) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(q + (static_cast<size_t>(w) * kPooled + g) * kC) + lane);
    const float a = warp_sum(fmaf(go.w, v.w, fmaf(go.z, v.z, fmaf(go.y, v.y, go.x * v.x))));
    if (lane == 0) s_ga[g] = a;
  }
  __syncthreads();
  float dot = 0.f;
  for (int g = tid; g < kPooled; g += 256) dot = fmaf(s_al[g], s_ga[g], dot);
  dot = warp_sum(dot);
  if (lane == 0) s_red[warp] = dot;
  __syncthreads();
  dot = ((s_red[0] + s_red[1]) + (s_red[2] + s_red[3])) + ((s_red[4] + s_red[5]) + (s_red[6] + s_red[7]));
  for (int g = tid; g < kLogitsLd; g += 256) {
    const size_t o = static_cast<size_t>(w) * kLogitsLd + g;
    alpha_out[o] = g < kPooled ? s_al[g] : 0.f;
    g_logit[o] = g < kPooled ? s_al[g] * (s_ga[g] - dot) : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------ IGLOO: g_y
// grid (94 position blocks, n), 256 threads; warp v handles pool group 8 b + v of the block, i.e. positions 8 (8 b + v) + r.
// Lane l holds output channels 4 l .. 4 l + 3.
//   value path: for each row r, the channels c routed to it (ballots over c = lane + 32 i: ascending c), acc += g_q[c] w_v^T[c]
//   patch path: the patch entries on the position (slots pos_start[t] .. pos_start[t+1] of the position-sorted packing, in
//               slot order), acc += g_mpi[patch] * 32 * ent_w[slot]   (ent_w holds Wf / 32, api.cu pack_patches)
// kLast = 1 (IGLOO#1 on y3): g_z3 = g_y3 * lrelu'(y3) to fp32 rows, and the block's max |g_z3| to blockmax[w][b];
// kLast = 0 (IGLOO#0 on y1): g_y1 to fp32 rows (conv2's backward epilogue adds it and applies the mask).
struct IglooBwdParams {
  const float* alpha;          // [n][752]
  const float* g_out;          // [n][256] (already offset to this IGLOO kernel's 128 columns)
  const uint8_t* route;        // [n][749][128]
  const float* wvT;            // [128 c][128 k]
  const float* g_mpi;          // [n][2100]
  const int32_t* pos_start;    // [5998] CSR over positions into the sorted entry slots
  const int32_t* slot_patch;   // [8400] patch index of every entry slot
  const float* ent_w;          // [slots][128]
  const uint8_t* y_rows;       // kLast: y3 activation rows (mask)
  float* out;                  // [n][5997][128]
  float* blockmax;             // kLast: [n][94]
};

template <bool kLast>
__global__ void __launch_bounds__(256)
attr_igloo_backward_kernel(const IglooBwdParams P) {
  __shared__ float s_gq[8][kC];
  __shared__ float s_max[8];
  const int w = blockIdx.y, b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int pg = b * 8 + warp;                                   // pool group of this warp
  const float4* wvT4 = reinterpret_cast<const float4*>(P.wvT);
  const float4* ew4 = reinterpret_cast<const float4*>(P.ent_w);
  float amax = 0.f;
  uint32_t rt[4] = {0u, 0u, 0u, 0u};
  if (pg < kPooled) {
    const float al = P.alpha[static_cast<size_t>(w) * kLogitsLd + pg];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = lane + 32 * i;
      s_gq[warp][c] = al * P.g_out[static_cast<size_t>(w) * 256 + c];
      rt[i] = P.route[(static_cast<size_t>(w) * kPooled + pg) * kC + c];
    }
  }
  __syncwarp();
  for (int r = 0; r < kPool; ++r) {
    const int t = pg * kPool + r;
    if (t >= kTok) break;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pg < kPooled) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t msk = __ballot_sync(0xffffffffu, rt[i] == static_cast<uint32_t>(r));
        while (msk) {
          const int c = 32 * i + __ffs(msk) - 1;
          msk &= msk - 1;
          const float gq = s_gq[warp][c];
          const float4 v = __ldg(wvT4 + c * (kC / 4) + lane);
          acc.x = fmaf(gq, v.x, acc.x); acc.y = fmaf(gq, v.y, acc.y); acc.z = fmaf(gq, v.z, acc.z); acc.w = fmaf(gq, v.w, acc.w);
        }
      }
    }
    const int e1 = P.pos_start[t + 1];
    for (int e = P.pos_start[t]; e < e1; ++e) {
      const float gm = kActScale * P.g_mpi[static_cast<size_t>(w) * kPatches + P.slot_patch[e]];
      const float4 v = __ldg(ew4 + static_cast<size_t>(e) * (kC / 4) + lane);
      acc.x = fmaf(gm, v.x, acc.x); acc.y = fmaf(gm, v.y, acc.y); acc.z = fmaf(gm, v.z, acc.z); acc.w = fmaf(gm, v.w, acc.w);
    }
    const size_t row = static_cast<size_t>(w) * kTok + t;
    if (kLast) {
      const __half2* yh = reinterpret_cast<const __half2*>(P.y_rows + row * kRowBytes + kOffHi16) + 2 * lane;
      const float2 y01 = __half22float2(yh[0]), y23 = __half22float2(yh[1]);
      acc.x = y01.x > 0.f ? acc.x : acc.x * kLeaky; acc.y = y01.y > 0.f ? acc.y : acc.y * kLeaky;
      acc.z = y23.x > 0.f ? acc.z : acc.z * kLeaky; acc.w = y23.y > 0.f ? acc.w : acc.w * kLeaky;
      amax = fmaxf(amax, fmaxf(fmaxf(fabsf(acc.x), fabsf(acc.y)), fmaxf(fabsf(acc.z), fabsf(acc.w))));
    }
    reinterpret_cast<float4*>(P.out + row * kC)[lane] = acc;
  }
  if (kLast) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
    if (lane == 0) s_max[warp] = amax;
    __syncthreads();
    if (tid == 0) {
      float m = s_max[0];
      for (int i = 1; i < 8; ++i) m = fmaxf(m, s_max[i]);
      P.blockmax[static_cast<size_t>(w) * kAttrPosBlocks + b] = m;
    }
  }
}

// 2^k with gmax * 2^k in [2^(top-1), 2^top) (1 for an all-zero gradient)
__device__ __forceinline__ float attr_scale_of(float gmax, int top) {
  if (!(gmax > 0.f) || !isfinite(gmax)) return 1.f;
  int e;
  frexpf(gmax, &e);                                              // gmax = m 2^e, m in [0.5, 1)
  return ldexpf(1.f, max(-120, min(120, top - e)));
}

// fp32 gradient rows (natural order) -> conv operand rows (hi16 | - | e4m3 pairs) of s * g at row 5996 - t, the input of a
// conv's backward pass, with s the per-window power of two that puts max |g| s in [2^(kTop-1), 2^kTop).  s depends only on the
// window's maximum (kNb block maxima of |g| per window), so s times the rows is the same bits for any gradient scale.
// grid (24, n), 256 threads, one warp per position; block 0 also stores s.  With `status`, a window whose scaled maximum lies
// above the hi8 plane's range (a gradient that is not finite) raises act_overflow, stage 0.
template <int kNb, int kTop>
__device__ __forceinline__ void attr_pack_body(const float* __restrict__ g, const float* __restrict__ blockmax,
                                               float* __restrict__ s_out, uint8_t* __restrict__ rows_out, DeviceStatus* status) {
  __shared__ float s_sw;
  const int w = blockIdx.y, t0 = blockIdx.x * kAttrSeg, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    float m = 0.f;
    for (int i = 0; i < kNb; ++i) m = fmaxf(m, blockmax[static_cast<size_t>(w) * kNb + i]);
    s_sw = attr_scale_of(m, kTop);
    if (blockIdx.x == 0) {
      s_out[w] = s_sw;
      if (status && !(m * s_sw <= kHi8Limit / kActScale)) { status->act_overflow = 1; status->ov_stage[0] = 1; }
    }
  }
  __syncthreads();
  const float sc = kActScale * s_sw;
  const int i_end = min(kAttrSeg, kTok - t0);
  for (int i = warp; i < i_end; i += 8) {
    const int t = t0 + i;
    float4 a = reinterpret_cast<const float4*>(g + (static_cast<size_t>(w) * kTok + t) * kC)[lane];
    a.x *= sc; a.y *= sc; a.z *= sc; a.w *= sc;
    __half2 h01, h23, l01, l23;
    split2_f16(a.x, a.y, h01, l01);
    split2_f16(a.z, a.w, h23, l23);
    const float2 fa = __half22float2(h01), fb = __half22float2(h23);
    uint8_t* rowp = rows_out + (static_cast<size_t>(w) * kTok + (kTok - 1 - t)) * kRowBytes;
    *reinterpret_cast<uint2*>(rowp + kOffHi16 + lane * 8) =
        make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
    *reinterpret_cast<uint2*>(rowp + kOffP8 + lane * 8) = make_uint2(
        static_cast<uint32_t>(pack_e4m3x2((a.x - fa.x) * kLo8Scale, fa.x * kHi8Scale)) |
            (static_cast<uint32_t>(pack_e4m3x2((a.y - fa.y) * kLo8Scale, fa.y * kHi8Scale)) << 16),
        static_cast<uint32_t>(pack_e4m3x2((a.z - fb.x) * kLo8Scale, fb.x * kHi8Scale)) |
            (static_cast<uint32_t>(pack_e4m3x2((a.w - fb.y) * kLo8Scale, fb.y * kHi8Scale)) << 16));
  }
}

// g_z3 (IGLOO#1's block maxima) -> s_w g_z3 rows, max |s_w g_z3| in [0.25, 0.5): the input of conv3's backward pass.  A
// gradient that is not finite reaches conv3's backward output and is reported by the g_z2 pack below.
__global__ void __launch_bounds__(256)
attr_pack_kernel(const float* __restrict__ g, const float* __restrict__ blockmax, float* __restrict__ s_w_out,
                 uint8_t* __restrict__ rows_out) {
  attr_pack_body<kAttrPosBlocks, -1>(g, blockmax, s_w_out, rows_out, nullptr);
}

// s_w g_z2 (conv3's backward output and its unit maxima) -> s2 s_w g_z2 rows, max in [1, 2): the input of conv2's backward pass
__global__ void __launch_bounds__(256)
attr_pack_gz2_kernel(const float* __restrict__ g, const float* __restrict__ unit_max, float* __restrict__ s2_out,
                     uint8_t* __restrict__ rows_out, DeviceStatus* status) {
  attr_pack_body<kUnitsPerWin * 8, 1>(g, unit_max, s2_out, rows_out, status);
}

// fp32 rows [n][5997][128] reversed in place within each window (gnm_debug_fetch of the time-reversed operand rows)
__global__ void reverse_rows_kernel(float* __restrict__ rows, int n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t half = static_cast<size_t>(kTok / 2) * kC;
  if (i >= static_cast<size_t>(n) * half) return;
  const size_t w = i / half, rc = i - w * half, r = rc / kC, c = rc - r * kC;
  float* a = rows + (w * kTok + r) * kC + c;
  float* b = rows + (w * kTok + (kTok - 1 - r)) * kC + c;
  const float t = *a;
  *a = *b;
  *b = t;
}

// ------------------------------------------------------------------------------------------------ layer 1
// attr[t] = (1 / s_w) sum_{u=t}^{min(t+5,5996)} <g_z1[u], W1[t-u+5, tok[t], :]>, tok from the window's bytes (token 0 = a
// 4-mer with a non-ACGT base, a real one-hot row).  grid (24, n), 256 threads, one warp per position, u ascending.
__global__ void __launch_bounds__(256)
layer1_attr_kernel(const uint8_t* __restrict__ ascii, const float* __restrict__ g_z1, const float* __restrict__ table,
                   const float* __restrict__ s_w, float* __restrict__ attr) {
  __shared__ int16_t s_tok[kAttrSeg];
  const int w = blockIdx.y, t0 = blockIdx.x * kAttrSeg, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  {
    const int t = t0 + threadIdx.x;
    if (t < kTok) {
      const uint8_t* s = ascii + static_cast<size_t>(w) * kWindow + t;
      s_tok[threadIdx.x] = static_cast<int16_t>(kmer_token(base_code(s[0]), base_code(s[1]), base_code(s[2]), base_code(s[3])));
    }
  }
  __syncthreads();
  const float inv = 1.f / s_w[w];
  const int i_end = min(kAttrSeg, kTok - t0);
  for (int i = warp; i < i_end; i += 8) {
    const int t = t0 + i, tk = s_tok[i];
    float a = 0.f;
    const int u_end = min(t + 5, kTok - 1);
    for (int u = t; u <= u_end; ++u) {
      const float4 gz = reinterpret_cast<const float4*>(g_z1 + (static_cast<size_t>(w) * kTok + u) * kC)[lane];
      const float4 wr = __ldg(reinterpret_cast<const float4*>(table + (static_cast<size_t>(t - u + 5) * kVocab + tk) * kC) + lane);
      a = fmaf(gz.w, wr.w, fmaf(gz.z, wr.z, fmaf(gz.y, wr.y, fmaf(gz.x, wr.x, a))));
    }
    a = warp_sum(a);
    if (lane == 0) attr[static_cast<size_t>(w) * kTok + t] = a * inv;
  }
}

// ------------------------------------------------------------------------------------------------ integrated gradients
// Layer 1 of row r of an integrated-gradients chunk: window r / m at alpha_k (encode.cuh, ig_row).  The gradient of log p_c at
// x' + alpha (x - x') with respect to the one-hot input is g[t, v] = (1 / s_w) sum_u <g_z1[u], W1[t-u+5, v, :]> at any v, so
//   zero baseline: out[r][t] = g[t, tok[t]]                   (x - x' = the one-hot row of tok[t])
//   N baseline:    out[r][t] = g[t, tok[t]] - g[t, 0]         (x - x' = e_tok - e_0; 0 where tok[t] = 0)
// each dot product in layer1_attr_kernel's order, so g[t, tok[t]] is bitwise what that kernel computes for the row.
// grid (24, rows), 256 threads, one warp per position, u ascending.  out: [rows][5997] (the workspace's g_y1 rows, free once
// conv2's backward has consumed them).
__global__ void __launch_bounds__(256)
layer1_ig_kernel(const uint8_t* __restrict__ ascii, const float* __restrict__ g_z1, const float* __restrict__ table,
                 const float* __restrict__ s_w, int m, int baseline, float* __restrict__ out) {
  __shared__ int16_t s_tok[kAttrSeg];
  const int r = blockIdx.y, t0 = blockIdx.x * kAttrSeg, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w = ig_row(r, m).win;
  {
    const int t = t0 + threadIdx.x;
    if (t < kTok) {
      const uint8_t* s = ascii + static_cast<size_t>(w) * kWindow + t;
      s_tok[threadIdx.x] = static_cast<int16_t>(kmer_token(base_code(s[0]), base_code(s[1]), base_code(s[2]), base_code(s[3])));
    }
  }
  __syncthreads();
  const float inv = 1.f / s_w[r];
  const bool sub = baseline == kIgN;
  const int i_end = min(kAttrSeg, kTok - t0);
  for (int i = warp; i < i_end; i += 8) {
    const int t = t0 + i, tk = s_tok[i];
    if (sub && tk == 0) {                                        // x - x' = 0 at this position
      if (lane == 0) out[static_cast<size_t>(r) * kTok + t] = 0.f;
      continue;
    }
    float a = 0.f, a0 = 0.f;
    const int u_end = min(t + 5, kTok - 1);
    for (int u = t; u <= u_end; ++u) {
      const float4 gz = reinterpret_cast<const float4*>(g_z1 + (static_cast<size_t>(r) * kTok + u) * kC)[lane];
      const float4 wr = __ldg(reinterpret_cast<const float4*>(table + (static_cast<size_t>(t - u + 5) * kVocab + tk) * kC) + lane);
      a = fmaf(gz.w, wr.w, fmaf(gz.z, wr.z, fmaf(gz.y, wr.y, fmaf(gz.x, wr.x, a))));
      if (sub) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(table + static_cast<size_t>(t - u + 5) * kVocab * kC) + lane);
        a0 = fmaf(gz.w, w0.w, fmaf(gz.z, w0.z, fmaf(gz.y, w0.y, fmaf(gz.x, w0.x, a0))));
      }
    }
    a = warp_sum(a);
    if (sub) a = a * inv - warp_sum(a0) * inv;
    else a *= inv;
    if (lane == 0) out[static_cast<size_t>(r) * kTok + t] = a;
  }
}

// IG[w][t] = (((g_0 + g_1) + g_2) + ... + g_{m-1}) / m over rows w m + k of layer1_ig_kernel, k ascending, fp32, no atomics.
// grid (24, windows), 256 threads, one position per thread.
__global__ void __launch_bounds__(256)
ig_reduce_kernel(const float* __restrict__ rows, int m, float* __restrict__ out) {
  const int w = blockIdx.y, t = blockIdx.x * 256 + threadIdx.x;
  if (t >= kTok) return;
  const float* g = rows + static_cast<size_t>(w) * m * kTok + t;
  float a = g[0];
  for (int k = 1; k < m; ++k) a += g[static_cast<size_t>(k) * kTok];
  out[static_cast<size_t>(w) * kTok + t] = a / static_cast<float>(m);
}

// log p_c from a row of C fp32 probabilities without cancellation: -log1p(sum_{i != c} p_i) (the sum in ascending i, as the
// head gradient's) when c is the argmax (p_c >= every p_i), log p_c otherwise; evaluated in fp64 and rounded once to fp32.
// out[2 i] for i < n, from probs row i, or from row 0 for every i when `broadcast` (the baseline's value in every row).
__global__ void __launch_bounds__(256)
ig_logp_kernel(const float* __restrict__ probs, int broadcast, int n, int tc /* attr_classes(target, C) */,
               float* __restrict__ out) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const int target = attr_target_of(tc), C = attr_count_of(tc);
  const float* p = probs + (broadcast ? 0 : static_cast<size_t>(i) * C);
  float other = 0.f;
  bool top = true;
  for (int k = 0; k < C; ++k)
    if (k != target) { other += p[k]; top = top && p[target] >= p[k]; }
  out[static_cast<size_t>(i) * 2] = top ? static_cast<float>(-log1p(static_cast<double>(other)))
                                        : static_cast<float>(log(static_cast<double>(p[target])));
}

}  // namespace gnm
