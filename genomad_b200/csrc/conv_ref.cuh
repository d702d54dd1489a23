// fp32 CUDA-core versions of the conv / w_v stages.  These are VALIDATION kernels: they exist so
// the tensor-core path (conv_t.cuh) can be checked on the GPU against an independent, obviously
// correct implementation at batch sizes the CPU oracle cannot reach (option "conv_impl" = 1).
// They are not a fallback: the product path never selects them on its own.
//
// Reference semantics: genomad/neural_network/igloo.py:64-72 (conv + LeakyReLU), :208-210 (w_v, max-pool).
#pragma once
#include "common.cuh"

namespace gnm {

constexpr int kRefPos = 32;                 // positions per CTA
constexpr int kRefThreads = 256;
template <int kNTaps> constexpr int ref_smem_bytes() {
  return ((kRefPos + kNTaps - 1) * kC + kC * kC) * static_cast<int>(sizeof(float));
}

// out_f32[n][5997][128] = act( bias + sum_j x[t - (kNTaps-1) + j] @ W[j] ),  x = hi + lo of y_in rows.
// W: [kNTaps][128 in][128 out] fp32 (Keras layout).  kNTaps = 6 (conv) or 1 (w_v, no bias/act).
template <int kNTaps, bool kBiasAct>
__global__ void __launch_bounds__(kRefThreads)
conv_ref_kernel(const uint8_t* __restrict__ y_in, const float* __restrict__ W, const float* __restrict__ bias,
                float* __restrict__ out_f32) {
  extern __shared__ float s_ref[];
  float* s_x = s_ref;                                   // [(32 + taps - 1)][128]
  float* s_w = s_ref + (kRefPos + kNTaps - 1) * kC;     // [128][128]
  const int w = blockIdx.y;
  const int t0 = blockIdx.x * kRefPos;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < (kRefPos + kNTaps - 1) * kC; i += kRefThreads) {
    const int r = i / kC, c = i - r * kC;
    const int t = t0 - (kNTaps - 1) + r;
    float v = 0.f;
    if (t >= 0 && t < kTok) {
      const uint8_t* row = y_in + (static_cast<size_t>(w) * kTok + t) * kRowBytes;
      v = (__half2float(reinterpret_cast<const __half*>(row + kOffHi16)[c]) +
           __half2float(reinterpret_cast<const __half*>(row + kOffLo16)[c])) * (1.f / kActScale);
    }
    s_x[i] = v;
  }
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  for (int j = 0; j < kNTaps; ++j) {
    __syncthreads();
    for (int i = threadIdx.x; i < kC * kC / 4; i += kRefThreads)
      reinterpret_cast<float4*>(s_w)[i] = reinterpret_cast<const float4*>(W + static_cast<size_t>(j) * kC * kC)[i];
    __syncthreads();
    for (int ci = 0; ci < kC; ++ci) {
      const float4 wv = *reinterpret_cast<const float4*>(s_w + ci * kC + tx * 4);
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const float x = s_x[(ty * 4 + a + j) * kC + ci];
        acc[a][0] = fmaf(x, wv.x, acc[a][0]);
        acc[a][1] = fmaf(x, wv.y, acc[a][1]);
        acc[a][2] = fmaf(x, wv.z, acc[a][2]);
        acc[a][3] = fmaf(x, wv.w, acc[a][3]);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int t = t0 + ty * 4 + a;
    if (t >= kTok) continue;
    float4 o = make_float4(acc[a][0], acc[a][1], acc[a][2], acc[a][3]);
    if (kBiasAct) {
      const float4 b = *reinterpret_cast<const float4*>(bias + tx * 4);
      o.x = lrelu(o.x + b.x); o.y = lrelu(o.y + b.y); o.z = lrelu(o.z + b.z); o.w = lrelu(o.w + b.w);
    }
    *reinterpret_cast<float4*>(out_f32 + (static_cast<size_t>(w) * kTok + t) * kC + tx * 4) = o;
  }
}

// fp32 rows -> activation rows (hi16 / lo16 planes only: the validation kernels never read the fp8 planes)
__global__ void split_rows_kernel(const float* __restrict__ in_f32, uint8_t* __restrict__ y_out, size_t n_rows) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;   // one thread per (row, 4 channels)
  if (i >= n_rows * (kC / 4)) return;
  const size_t r = i / (kC / 4);
  const int c4 = static_cast<int>(i - r * (kC / 4));
  const float4 v = reinterpret_cast<const float4*>(in_f32)[i];
  __half h0, h1, h2, h3, l0, l1, l2, l3;
  split_f16(kActScale * v.x, h0, l0); split_f16(kActScale * v.y, h1, l1);
  split_f16(kActScale * v.z, h2, l2); split_f16(kActScale * v.w, h3, l3);
  uint8_t* row = y_out + r * kRowBytes;
  *reinterpret_cast<uint2*>(row + kOffHi16 + c4 * 8) = make_uint2(pack_h2(h0, h1), pack_h2(h2, h3));
  *reinterpret_cast<uint2*>(row + kOffLo16 + c4 * 8) = make_uint2(pack_h2(l0, l1), pack_h2(l2, l3));
}

// activation rows -> fp32 rows (debug fetch): (hi16 + lo16) / 32, or (hi16 + lo8 / 128) / 32 for rows written by
// conv2 (which stores only the planes conv3 reads)
__global__ void join_rows_kernel(const uint8_t* __restrict__ y_in, float* __restrict__ out_f32, size_t n_rows, int fp8_lo) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_rows * kC) return;
  const size_t r = i / kC;
  const int c = static_cast<int>(i - r * kC);
  const uint8_t* row = y_in + r * kRowBytes;
  const float hi = __half2float(reinterpret_cast<const __half*>(row + kOffHi16)[c]);
  float lo;
  if (fp8_lo) {
    const __half_raw hr = __nv_cvt_fp8_to_halfraw(row[kOffP8 + 2 * c], __NV_E4M3);        // pair (lo8[c], hi8[c])
    lo = __half2float(__half(hr)) * (1.f / kLo8Scale);
  } else {
    lo = __half2float(reinterpret_cast<const __half*>(row + kOffLo16)[c]);
  }
  out_f32[i] = (hi + lo) * (1.f / kActScale);
}

// z[n][5997][128] -> q[n][749][128] = max over 8 consecutive positions (valid pooling)
__global__ void maxpool8_kernel(const float* __restrict__ z, float* __restrict__ q, int n_windows) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t total = static_cast<size_t>(n_windows) * kPooled * kC;
  if (i >= total) return;
  const int c = static_cast<int>(i % kC);
  const size_t wg = i / kC;
  const int g = static_cast<int>(wg % kPooled);
  const size_t w = wg / kPooled;
  const float* src = z + (w * kTok + static_cast<size_t>(g) * kPool) * kC + c;
  float m = src[0];
#pragma unroll
  for (int r = 1; r < kPool; ++r) m = fmaxf(m, src[static_cast<size_t>(r) * kC]);
  q[i] = m;
}

}  // namespace gnm
