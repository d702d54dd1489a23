// libgnm.so -- C ABI (include/gnm.h) over the sm_90a kernels of the geNomad nn-classification path.
// Host side of the library: weight re-packing, workspace, TMA descriptors, stage orchestration.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/gnm.h"
#include "common.cuh"
#include "encode.cuh"
#include "conv_t.cuh"
#include "layer1_wv.cuh"
#include "conv_ref.cuh"
#include "igloo.cuh"
#include "dense.cuh"
#include "logits_tc.cuh"
#include "wv_gather.cuh"
#include "contigs.cuh"
#include "attr.cuh"
#include "neighbours.cuh"
#include "clusters.cuh"
#include "head.cuh"
#include "regions.cuh"
#include "novelty.cuh"
#include "layout.cuh"
#include "ivf.cuh"

using namespace gnm;

// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int fail(const std::string& m) { g_err = m; return 1; }

#define GNM_CUDA(expr)                                                                       \
  do {                                                                                       \
    cudaError_t e__ = (expr);                                                                \
    if (e__ != cudaSuccess)                                                                  \
      return fail(std::string(#expr) + " failed: " + cudaGetErrorString(e__) + " (" __FILE__ \
                  ":" + std::to_string(__LINE__) + ")");                                     \
  } while (0)

extern "C" const char* gnm_last_error(void) { return g_err.c_str(); }
extern "C" const char* gnm_version(void) { return "libgnm 0.4 (sm_90a; wgmma fp16 + e4m3 split convs, fused fp16x3 w_v + patch gather, tf32x3 logits and dense head)"; }

// ------------------------------------------------------------------------------------------------
struct StageTimer {
  std::vector<const char*> names;
  std::vector<cudaEvent_t> events;   // events[i] recorded BEFORE stage i; last one after the final stage
};

struct gnm_handle {
  int device = 0;
  int max_batch = 0;
  int num_sms = 0;
  long long launches = 0;
  // options
  int conv_impl = 0;        // 0 tensor cores (wgmma), 1 fp32 validation kernels
  int debug_stop = 0;       // 0 = full pipeline; 1 = stop after embed+gather0; 2 = after conv2; 3 = after conv3
  int profile_stages = 0;
  int conv_experiment = 0;
  int conv_cluster = 1;     // experiment: thread-block cluster size of the conv kernel's launch (1 = no clusters)
  int fuse_gather = 1;      // 1 = w_v + patch gather in one pass over the activations (wv_gather.cuh); 0 = conv_t_kernel<true> + patch_stream_kernel
  int fuse_l1 = 0;          // 1 = layer 1 and w_v#0 in one kernel (layer1_wv.cuh; bit-identical, measured slower: off); 0 = embed_conv1_kernel + conv_t_kernel<true>
  long long* conv_dbg = nullptr;                    // [num_sms][8] cycle counters of the last conv_t_kernel<false> launch
  // weights on device
  float* conv1_table = nullptr; float* conv1_triple = nullptr; float* conv1_bias = nullptr;
  uint8_t* wpack[4] = {nullptr, nullptr, nullptr, nullptr};  // conv2, conv3, w_v#0, w_v#1 -- 16 KB TMA stages in consumption order
  float conv_out_scale[2] = {1.f, 1.f};             // 2^-S per conv layer (see conv_t.cuh)
  float* conv_bias[2] = {nullptr, nullptr};
  float* conv_w32[2] = {nullptr, nullptr};          // Keras layout fp32 (validation kernels)
  float* wv32[2] = {nullptr, nullptr};
  float* ent_w[2] = {nullptr, nullptr}; int32_t* ent_pos[2] = {nullptr, nullptr}; int32_t* slot_of[2] = {nullptr, nullptr};
  float* wbias[2] = {nullptr, nullptr}; float* wqk[2] = {nullptr, nullptr};
  float* d0w = nullptr; float* d0b = nullptr; float* bn0_scale = nullptr; float* bn0_shift = nullptr;
  float* d1w = nullptr; float* d1b = nullptr; float* bn1_scale = nullptr; float* bn1_shift = nullptr;
  float* d2w = nullptr; float* d2b = nullptr;
  // tensor-core head (3 x TF32, logits_tc_kernel): transposed weights [512][K] and the activations as TF32 halves
  float* dwT_hi[2] = {nullptr, nullptr}; float* dwT_lo[2] = {nullptr, nullptr};
  float* hA_hi[2] = {nullptr, nullptr}; float* hA_lo[2] = {nullptr, nullptr};       // h0 [mb][256], h1 [mb][512]
  CUtensorMap tm_hd_a[2][2]; CUtensorMap tm_hd_b[2][2];                              // [layer][hi/lo]
  // workspace
  uint8_t* ybuf[2] = {nullptr, nullptr};            // activation rows, 768 B per position
  int ybuf_fp8lo[2] = {0, 0};                        // 1 = the buffer was written by conv2 (hi16 + lo8 + hi8 only)
  float* q[2] = {nullptr, nullptr};
  float* mpi[2] = {nullptr, nullptr};
  float* mpi_hi[2] = {nullptr, nullptr}; float* mpi_lo[2] = {nullptr, nullptr};   // TF32 halves of mpi (logits_tc.cuh)
  float* wqkT_hi[2] = {nullptr, nullptr}; float* wqkT_lo[2] = {nullptr, nullptr}; // TF32 halves of w_qk^T [749][2100]
  CUtensorMap tm_lg_a[2][2];                         // [igloo][hi/lo] over mpi_hi / mpi_lo
  CUtensorMap tm_lg_b[2][2];                         // [igloo][hi/lo] over wqkT_hi / wqkT_lo
  float* part = nullptr;                             // [max_batch][kGsSlots] per-entry partial dot products ([kGsSlots][mb_pad] in the fused path)
  int2* grp[2] = {nullptr, nullptr};                 // wv_gather_kernel: position groups {first entry slot, row in band | entries << 8}
  int32_t* band_gstart[2] = {nullptr, nullptr};      // [kNumBands + 1] first position group of every band
  uint4* wfrag[2] = {nullptr, nullptr};              // [kGsSlots][2][4][4] folded weights as mma.m16n8k16 B fragments (fp16 hi / lo halves)
  float gather_unscale[2] = {1.f, 1.f};              // 1 / the power of two applied to the folded weights before the fp16 split
  float wv_out_scale[2] = {1.f, 1.f};                // 2^-e / 32: undoes the power of two applied to w_v before its fp16 split
  std::vector<int32_t> band_groups[2];               // host copy: position groups per band (cost model of wv_gather_kernel's unit split)
  int32_t* cta_split = nullptr;                      // [num_sms + 1] device: unit range per CTA of the current launch
  std::vector<int32_t> split_host[2];                // host copy of the last split per IGLOO kernel (source of the async upload)
  int split_groups[2] = {-1, -1}, split_grid[2] = {-1, -1};
  // Unit cost model of wv_split: base + per position group of the busiest gather warp.  Fitted by least squares to the per-CTA
  // cycle counters of a batch-1024 launch (tools/ab_stages.py --wvg-fit: CTA cycles = a x units + b x summed busiest-warp groups,
  // 132 CTAs, 8 launches averaged; wv_cost_group = b / a).  H100, shipped patch sets: a = 7,912 and b = 254 cycles, so 0.032.
  // With the folded weights read per unit the same fit gave 0.164; keeping them in registers made a group ~4x cheaper.
  float wv_cost_base = 1.f, wv_cost_group = 0.032f;
  int mb_pad = 0;                                    // max_batch rounded up to a multiple of 8 (window groups of wv_gather_kernel)
  CUtensorMap tm_band[2];                            // activations, box = 128 B x 8 windows x 24 positions (make_band_map)
  float* logits = nullptr; float* logits_part = nullptr; float* h0 = nullptr; float* h1 = nullptr; float* h2 = nullptr;
  float* scratch32 = nullptr;                        // validation path only, allocated lazily
  uint8_t* in_stage[2] = {nullptr, nullptr};         // gnm_classify_host
  float* out_stage[2] = {nullptr, nullptr};
  // second set of the buffers that a step's main part writes and its tail reads (q, mpi + TF32 halves): with two sets the tail
  // of step i (logits / attention / head, on tail_stream) overlaps the main part of step i+1 (tail_overlap, see forward_many)
  float* q_set[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};
  float* mpi_set[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};
  float* mpi_hi_set[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};
  float* mpi_lo_set[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};
  CUtensorMap tm_lg_a_set[2][2][2];                  // [parity][igloo][hi/lo]
  int tail_overlap = 1;                              // option: 1 = overlap (multi-step calls only), 0 = strictly in order
  cudaStream_t tail_stream = nullptr;
  cudaEvent_t main_done[2] = {nullptr, nullptr}, tail_done[2] = {nullptr, nullptr};
  cudaStream_t copy_stream = nullptr, compute_stream = nullptr;
  cudaEvent_t in_ready[2] = {nullptr, nullptr}, in_free[2] = {nullptr, nullptr};
  DeviceStatus* status = nullptr;                    // pinned host memory, device-visible
  CUtensorMap tm_act[2];
  CUtensorMap tm_w[4];                               // weight packs, one 16 KB stage per box
  CUtensorMap tm_w_half[4];                          // the same packs, one warpgroup's 8 KB half-stage per box (conv_t_kernel)
  StageTimer timer;
  std::vector<void*> allocs;
  const uint8_t* attr_route[2] = {nullptr, nullptr};   // routing / maxima of the last attribution chunk (gnm_debug_fetch "route*", "routeq*")
  const float* attr_rq[2] = {nullptr, nullptr};
  const gnm_attr* attr_last = nullptr;                 // the context of the last attribution chunk (gnm_debug_fetch "attr_*")
  int attr_mb = 0;                                     // max_batch of the context those buffers belong to
};

// ------------------------------------------------------------------------------------------------
template <class O, class T>     // O: any owner with an `allocs` list (the handle, a head, a trainer)
static int dev_upload(O* h, T** dst, const T* src, size_t count) {
  GNM_CUDA(cudaMalloc(reinterpret_cast<void**>(dst), count * sizeof(T)));
  h->allocs.push_back(*dst);
  GNM_CUDA(cudaMemcpy(*dst, src, count * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}
template <class O, class T>
static int dev_alloc(O* h, T** dst, size_t count) {
  GNM_CUDA(cudaMalloc(reinterpret_cast<void**>(dst), count * sizeof(T)));
  h->allocs.push_back(*dst);
  return 0;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int get_encode_fn(PFN_encodeTiled* fn) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  GNM_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || !p) return fail("cuTensorMapEncodeTiled not available from the driver");
  *fn = reinterpret_cast<PFN_encodeTiled>(p);
  return 0;
}

// activations [n][5997][768 B] viewed as bytes; box = 128 bytes (one plane slice) x 136 rows x 1 window, 128B swizzle,
// rows outside [0, 5997) read as 0 (= causal padding)
static int make_act_map(PFN_encodeTiled enc, CUtensorMap* tm, uint8_t* base, int n_windows, int box_rows = kSlabRows) {
  cuuint64_t dims[3] = {kRowBytes, kTok, static_cast<cuuint64_t>(n_windows)};
  cuuint64_t strides[2] = {kRowBytes, static_cast<cuuint64_t>(kTok) * kRowBytes};
  cuuint32_t box[3] = {128, static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled(activations) failed: " + std::to_string(int(r)));
  return 0;
}
// wv_gather_kernel's view of the activations: the WINDOW axis is listed before the POSITION axis (strides need not ascend), so
// the box {128 B, 8 windows, 24 positions} lands in shared memory as [position][window][128 B]: the 8 windows of one position are
// one 1024-byte swizzle atom -- what the gather's ldmatrix wants -- and the 192 rows are still one K-major wgmma operand.
static int make_band_map(PFN_encodeTiled enc, CUtensorMap* tm, uint8_t* base, int n_windows) {
  cuuint64_t dims[3] = {kRowBytes, static_cast<cuuint64_t>(n_windows), kTok};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(kTok) * kRowBytes, kRowBytes};
  cuuint32_t box[3] = {128, kBandWins, kBandRows};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled(activation bands) failed: " + std::to_string(int(r)));
  return 0;
}
// packed weights [stages*128 rows][128 B]; box = 128 B x box_rows
static int make_w_map(PFN_encodeTiled enc, CUtensorMap* tm, uint8_t* base, int n_stages, int box_rows) {
  cuuint64_t dims[2] = {128, static_cast<cuuint64_t>(n_stages) * 128};
  cuuint64_t strides[1] = {128};
  cuuint32_t box[2] = {128, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled(weights) failed: " + std::to_string(int(r)));
  return 0;
}

// fp32 matrix [rows][inner] (row pitch = inner * 4 B), box = 32 floats (128 B) x box_rows, 128B swizzle, OOB -> 0
static int make_f32_map(PFN_encodeTiled enc, CUtensorMap* tm, float* base, int inner, int rows, int box_rows) {
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(inner) * sizeof(float)};
  cuuint32_t box[2] = {32, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled(fp32 matrix) failed: " + std::to_string(int(r)));
  return 0;
}

// One 16 KB fp16 TMA stage: B[n][kk] = fp16(part(W[k = kh*64 + kk][n] * scale)), part = hi or lo of the fp16 split.  The split
// is taken of the scaled weight (scale is a power of two), so weights far below 1 keep their precision instead of falling into
// fp16's subnormal range.
static void pack_stage_f16(std::vector<uint8_t>& dst, const float* Wkn /* [128 k][128 n] */, int w_lo, int kh, float scale) {
  for (int n = 0; n < kC; ++n)
    for (int kk = 0; kk < 64; ++kk) {
      const float x = Wkn[static_cast<size_t>(kh * 64 + kk) * kC + n] * scale;
      const __half hi = __float2half_rn(x);
      const float v = w_lo ? x - __half2float(hi) : __half2float(hi);
      const uint16_t bits = __half_as_ushort(__float2half_rn(v));
      dst.push_back(static_cast<uint8_t>(bits & 0xff));
      dst.push_back(static_cast<uint8_t>(bits >> 8));
    }
}
// One 16 KB e4m3 TMA stage of the correction passes: B[n][2c + s] for the 64 input channels c of K-half kh, interleaved like the
// activation pairs (common.cuh): with x = W * scale split into hi = fp16(x) and lo = x - hi (the main pass's split),
// s = 0 multiplies lo8(A) -> e4m3(hi * scale_hi), s = 1 multiplies hi8(A) -> e4m3(lo * scale_lo).
static void pack_stage_f8_pairs(std::vector<uint8_t>& dst, const float* Wkn, int kh, float scale, float scale_hi, float scale_lo) {
  for (int n = 0; n < kC; ++n)
    for (int c = 0; c < 64; ++c) {
      const float x = Wkn[static_cast<size_t>(kh * 64 + c) * kC + n] * scale;
      const float hi = __half2float(__float2half_rn(x));
      dst.push_back(static_cast<uint8_t>(__nv_cvt_float_to_fp8(hi * scale_hi, __NV_SATFINITE, __NV_E4M3)));
      dst.push_back(static_cast<uint8_t>(__nv_cvt_float_to_fp8((x - hi) * scale_lo, __NV_SATFINITE, __NV_E4M3)));
    }
}

// A conv layer's tensor-core weight pack, in the order conv_t_kernel consumes its 16 KB stages, and its output scale 2^-S.
// Wk: Keras layout [6 taps][128 in][128 out].  Common scale 2^S of the three passes (conv_t.cuh): main weights fp16(W * 2^d)
// with wmax * 2^d in (0.39, 0.78] * 2^16, so the fp16 plane and both e4m3 planes (|hi| * 2^-7 <= 400 < 448) stay in range.
// Small weights get d > 16: with d fixed at 16 the e4m3 plane of their lo halves fell into the subnormal range and the
// Ahi * Wlo correction stopped correcting.
static int pack_conv_weights(const float* Wk, std::vector<uint8_t>& pk, float* out_scale, const char* who) {
  float wmax = 0.f;
  for (size_t i = 0; i < static_cast<size_t>(kTaps) * kC * kC; ++i) wmax = std::max(wmax, std::fabs(Wk[i]));
  if (!(wmax > 0.f) || !std::isfinite(wmax)) return fail(std::string(who) + ": conv kernel is all-zero or not finite");
  const int shift = static_cast<int>(std::ceil(std::log2(wmax / 0.78f)));
  const int d = std::min(16 - shift, 40), S = 5 + d;
  if (d < 1) return fail(std::string(who) + ": conv weights too large for the fp16 operand format");
  *out_scale = std::ldexp(1.f, -S);
  pk.clear();                                           // (region, tap): hi16.k0 x6, hi16.k1 x6, pairs.k0 x6, pairs.k1 x6
  pk.reserve(static_cast<size_t>(kConvStages) * kBStage);
  for (int kh = 0; kh < 2; ++kh)
    for (int tap = 0; tap < kTaps; ++tap)
      pack_stage_f16(pk, Wk + static_cast<size_t>(tap) * kC * kC, 0, kh, std::ldexp(1.f, d));
  for (int kh = 0; kh < 2; ++kh)                        // x (lo8, hi8) = (e4m3(Alo * 2^12), e4m3(Ahi * 2^7)):  (e4m3(Whi * 2^(S-12)), e4m3(Wlo * 2^(S-7)))
    for (int tap = 0; tap < kTaps; ++tap)                //   = (e4m3(hi * 2^(S-12-d)), e4m3(lo * 2^(S-7-d))) of the split of W * 2^d
      pack_stage_f8_pairs(pk, Wk + static_cast<size_t>(tap) * kC * kC, kh, std::ldexp(1.f, d), std::ldexp(1.f, S - 12 - d),
                          std::ldexp(1.f, S - 7 - d));
  return 0;
}

// Exponent k of the power of two applied to w_v and to the folded patch weights before their fp16 hi / lo split: max |w| * 2^k
// in [2^13, 2^14), so that the lo halves stay in fp16's normal range.  k is clamped to [-126, 121], where 2^k, 2^-k (the
// gather's unscale) and 2^-k / 32 (the q epilogues' scale) are normal fp32: every max |w| >= 2^-107 gets its exact k, smaller
// ones keep k = 121 (their halves still carry the gather's precision while max |w| is a normal fp32 number), and no finite
// weight overflows the fp16 halves (max |w| < 2^128 needs k >= -114).  False if a weight is not finite: it has no split.
static constexpr int kSplitExpMin = -126, kSplitExpMax = 121;
static bool split_exponent(const float* w, size_t n, int* k) {
  float wmax = 0.f;
  for (size_t i = 0; i < n; ++i) {
    if (!std::isfinite(w[i])) return false;
    wmax = std::max(wmax, std::fabs(w[i]));
  }
  *k = 0;
  if (wmax > 0.f) { int ex; std::frexp(wmax, &ex); *k = std::max(kSplitExpMin, std::min(kSplitExpMax, 14 - ex)); }
  return true;
}

// One IGLOO layer's patch set as the gather kernels want it (host only).
//   * fold the patch weights (Wf = w_mult * w_summer / 32, reference igloo.py:199-204 applied to rows that carry the activation
//     scale), sort the 8,400 (patch, slot) entries by position and deal them to the kGsSlots entry slots (padding slots:
//     position 0, zero weights): ent_w / ent_pos / slot_of -- patch_stream_kernel's and patch_finish*'s view;
//   * wv_gather_kernel's view of the same sorted entries: POSITION GROUPS = the entries that sit on one position, at most
//     kWgGroupMax = 4 per group (the 8 columns of the warp-level mma are 4 entries x (hi, lo); 8,400 entries hit ~4,500 positions),
//     the first group of every band of kBandRows positions, and the folded weights as that instruction's B fragments: fp16 hi / lo
//     halves of w * 2^k (k = split_exponent; the kernel multiplies the sums by unscale = 2^-k).  Fragment word order per slot:
//     [K-half][k-step][tig] x {hi b0, hi b1, lo b0, lo b1}, b0 = channels (k0, k0 + 1), b1 = (k0 + 8, k0 + 9),
//     k0 = 64 K-half + 16 k-step + 2 tig.
// Returns false, with o incomplete, if a folded weight is not finite.
struct PatchPack {
  std::vector<float> ent_w;              // [kGsSlots][128]
  std::vector<int32_t> ent_pos, slot_of; // [kGsSlots], [8400]
  std::vector<int2> groups;              // {first slot, row inside the band | entries << 8}
  std::vector<int32_t> band_gstart;      // [kNumBands + 1]
  std::vector<uint32_t> frag;            // [kGsSlots][128]
  float unscale = 1.f;
};
static bool pack_patches(const int32_t* patches, const float* w_mult, const float* w_summer, PatchPack& o) {
  std::vector<int> order(static_cast<size_t>(kPatches) * kPatchLen);
  for (size_t i = 0; i < order.size(); ++i) order[i] = static_cast<int>(i);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return patches[a] < patches[b]; });
  o.ent_w.assign(static_cast<size_t>(kGsSlots) * kC, 0.f);
  o.ent_pos.assign(kGsSlots, 0);
  o.slot_of.assign(static_cast<size_t>(kPatches) * kPatchLen, 0);
  std::vector<float>& ent_w = o.ent_w;
  std::vector<int32_t>& ent_pos = o.ent_pos;
  for (size_t slot = 0; slot < order.size(); ++slot) {
    const int e = order[slot], k = e % kPatchLen;
    ent_pos[slot] = patches[e];
    o.slot_of[e] = static_cast<int32_t>(slot);
    for (int c = 0; c < kC; ++c)
      ent_w[slot * kC + c] = (w_mult[static_cast<size_t>(e) * kC + c] * w_summer[k * kC + c]) * (1.f / kActScale);
  }
  int k2;
  if (!split_exponent(ent_w.data(), ent_w.size(), &k2)) return false;
  const float wscale = std::ldexp(1.f, k2);
  o.unscale = std::ldexp(1.f, -k2);
  o.groups.clear();
  o.band_gstart.assign(kNumBands + 1, 0);
  const size_t n_ent = order.size();
  size_t slot = 0;
  for (int b = 0; b < kNumBands; ++b) {
    o.band_gstart[b] = static_cast<int32_t>(o.groups.size());
    while (slot < n_ent && ent_pos[slot] < (b + 1) * kBandRows) {
      size_t run = slot;
      while (run < n_ent && ent_pos[run] == ent_pos[slot] && run - slot < static_cast<size_t>(kWgGroupMax)) ++run;
      o.groups.push_back(make_int2(static_cast<int>(slot), (ent_pos[slot] - b * kBandRows) | (static_cast<int>(run - slot) << 8)));
      slot = run;
    }
  }
  o.band_gstart[kNumBands] = static_cast<int32_t>(o.groups.size());
  if (o.groups.empty()) o.groups.push_back(make_int2(0, 0));
  auto h2 = [](float x, float y) {
    return static_cast<uint32_t>(__half_as_ushort(__float2half_rn(x))) | (static_cast<uint32_t>(__half_as_ushort(__float2half_rn(y))) << 16);
  };
  o.frag.assign(static_cast<size_t>(kGsSlots) * 128, 0u);      // 512 B per entry slot
  for (size_t e = 0; e < n_ent; ++e)
    for (int kh = 0; kh < 2; ++kh)
      for (int ks = 0; ks < 4; ++ks)
        for (int tig = 0; tig < 4; ++tig) {
          const int k0 = kh * 64 + ks * 16 + 2 * tig;
          const int kk[4] = {k0, k0 + 1, k0 + 8, k0 + 9};
          float hi[4], lo[4];
          for (int i = 0; i < 4; ++i) {
            const float x = ent_w[e * kC + kk[i]] * wscale;
            hi[i] = __half2float(__float2half_rn(x));
            lo[i] = x - hi[i];
          }
          uint32_t* f = &o.frag[(((e * 2 + kh) * 4 + ks) * 4 + tig) * 4];
          f[0] = h2(hi[0], hi[1]); f[1] = h2(hi[2], hi[3]); f[2] = h2(lo[0], lo[1]); f[3] = h2(lo[2], lo[3]);
        }
  return true;
}
// Test hook (host only): the packing above for one IGLOO layer, into caller-owned buffers; see include/gnm.h.
extern "C" int gnm_pack_patches(const int32_t* patches, const float* w_mult, const float* w_summer, int32_t* slot_of, int32_t* ent_pos,
                                float* ent_w, int32_t* groups, int* n_groups, int32_t* band_first_group, uint32_t* frag, float* unscale,
                                int* layout) {
  if (layout) { layout[0] = kBandRows; layout[1] = kNumBands; layout[2] = kGsSlots; layout[3] = kWgGroupMax; }
  if (!patches && !w_mult && !w_summer) return 0;                       // layout query only
  if (!patches || !w_mult || !w_summer || !n_groups) return fail("gnm_pack_patches: null argument");
  for (int i = 0; i < kPatches * kPatchLen; ++i)
    if (patches[i] < 0 || patches[i] >= kTok) return fail("gnm_pack_patches: patch index out of range");
  PatchPack pk;
  if (!pack_patches(patches, w_mult, w_summer, pk))
    return fail("gnm_pack_patches: folded patch weights w_mult * w_summer / 32 not finite: no fp16 operand split carries them");
  const int real_groups = pk.band_gstart[kNumBands];
  if (groups && *n_groups < real_groups) return fail("gnm_pack_patches: groups buffer too small");
  if (slot_of) std::memcpy(slot_of, pk.slot_of.data(), pk.slot_of.size() * sizeof(int32_t));
  if (ent_pos) std::memcpy(ent_pos, pk.ent_pos.data(), pk.ent_pos.size() * sizeof(int32_t));
  if (ent_w) std::memcpy(ent_w, pk.ent_w.data(), pk.ent_w.size() * sizeof(float));
  if (groups) for (int i = 0; i < real_groups; ++i) { groups[2 * i] = pk.groups[i].x; groups[2 * i + 1] = pk.groups[i].y; }
  *n_groups = real_groups;
  if (band_first_group) std::memcpy(band_first_group, pk.band_gstart.data(), pk.band_gstart.size() * sizeof(int32_t));
  if (frag) std::memcpy(frag, pk.frag.data(), pk.frag.size() * sizeof(uint32_t));
  if (unscale) *unscale = pk.unscale;
  return 0;
}

// keras BN inference form  x * inv + (beta - mean * inv),  inv = gamma * rsqrt(var + eps)
static void fold_bn(const gnm_bn_weights& b, std::vector<float>& sc, std::vector<float>& sh) {
  sc.resize(kHidden); sh.resize(kHidden);
  for (int i = 0; i < kHidden; ++i) {
    const float inv = b.gamma[i] * (1.0f / std::sqrt(b.moving_variance[i] + 1e-3f));
    sc[i] = inv;
    sh[i] = b.beta[i] - b.moving_mean[i] * inv;
  }
}

// W [K in][512 out] -> W^T [512][K] as two TF32 halves: the K-major B operand of logits_tc_kernel
static void split_dense_t(const float* w, int K, std::vector<float>& thi, std::vector<float>& tlo) {
  thi.resize(static_cast<size_t>(kHidden) * K); tlo.resize(thi.size());
  for (int k = 0; k < K; ++k)
    for (int n = 0; n < kHidden; ++n)
      split_tf32(w[static_cast<size_t>(k) * kHidden + n], thi[static_cast<size_t>(n) * K + k], tlo[static_cast<size_t>(n) * K + k]);
}

// ------------------------------------------------------------------------------------------------
extern "C" int gnm_create(int device, const gnm_weights* w, int max_batch, gnm_handle** out) {
  if (!w || !out) return fail("gnm_create: null argument");
  if (max_batch < 1 || max_batch > 32768) return fail("gnm_create: max_batch must be in [1, 32768]");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("gnm_create: no CUDA device available (libgnm has no CPU fallback)");
  if (device < 0 || device >= ndev) return fail("gnm_create: bad device index");
  cudaDeviceProp prop;
  GNM_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(std::string("gnm_create: device is sm_") + std::to_string(prop.major * 10 + prop.minor) +
                ", this library is built for sm_90a (H100) only");
  GNM_CUDA(cudaSetDevice(device));
  gnm_handle* h = new gnm_handle();
  h->device = device;
  h->max_batch = max_batch;
  h->num_sms = prop.multiProcessorCount;
  *out = h;   // so the caller can gnm_destroy() after a partial failure

  // ---- validate patch indices (a bad index would read out of bounds)
  for (int s = 0; s < 2; ++s)
    for (int i = 0; i < kPatches * kPatchLen; ++i)
      if (w->igloo[s].patches[i] < 0 || w->igloo[s].patches[i] >= kTok)
        return fail("gnm_create: patch index out of range [0, 5997)");

  // ---- first layer table + bias
  if (dev_upload(h, &h->conv1_table, w->conv1_kernel, static_cast<size_t>(kTaps) * kVocab * kC)) return 1;
  if (dev_upload(h, &h->conv1_bias, w->conv1_bias, kC)) return 1;
  {
    // "triple" tables of layer 1 (encode.cuh): A[code] = (W1[0][k0] + W1[1][k1]) + W1[2][k2] for the three 4-mers of a
    // 6-base word, B likewise with taps 3..5 -- same fp32 operation order as the kernel's fallback path.
    std::vector<float> tri(static_cast<size_t>(2) * kTriple * kC);
    for (int half = 0; half < 2; ++half)
      for (int code = 0; code < kTriple; ++code) {
        const int k0 = 1 + (code >> 4), k1 = 1 + ((code >> 2) & 255), k2 = 1 + (code & 255);
        const float* r0 = w->conv1_kernel + (static_cast<size_t>(3 * half + 0) * kVocab + k0) * kC;
        const float* r1 = w->conv1_kernel + (static_cast<size_t>(3 * half + 1) * kVocab + k1) * kC;
        const float* r2 = w->conv1_kernel + (static_cast<size_t>(3 * half + 2) * kVocab + k2) * kC;
        float* dst = tri.data() + (static_cast<size_t>(half) * kTriple + code) * kC;
        for (int c = 0; c < kC; ++c) dst[c] = (r0[c] + r1[c]) + r2[c];
      }
    if (dev_upload(h, &h->conv1_triple, tri.data(), tri.size())) return 1;
  }

  // ---- tensor-core weight packs, in the order conv_t_kernel consumes its 16 KB stages
  {
    const float* convw[2] = {w->conv2_kernel, w->conv3_kernel};
    for (int L = 0; L < 2; ++L) {
      std::vector<uint8_t> pk;
      if (pack_conv_weights(convw[L], pk, &h->conv_out_scale[L], "gnm_create")) return 1;
      if (dev_upload(h, &h->wpack[L], pk.data(), pk.size())) return 1;
      if (dev_upload(h, &h->conv_w32[L], convw[L], static_cast<size_t>(kTaps) * kC * kC)) return 1;
    }
    for (int s = 0; s < 2; ++s) {                          // w_v: (K-half, weight hi/lo) of the fp16 split of w_v * 2^e
      // e moves max |w_v| to [2^13, 2^14) (split_exponent, as for the patch weights): unscaled, the lo halves of small weights
      // (|w| < 0.125) fall into fp16's subnormal range and the Ahi * Wlo pass stops correcting.  The q epilogues multiply by
      // 2^-e / 32.
      int e;
      if (!split_exponent(w->igloo[s].w_v, static_cast<size_t>(kC) * kC, &e))
        return fail("gnm_create: IGLOO layer " + std::to_string(s) + ": w_v not finite: no fp16 operand split carries it");
      h->wv_out_scale[s] = std::ldexp(1.f / kActScale, -e);
      std::vector<uint8_t> pk;
      for (int kh = 0; kh < 2; ++kh)
        for (int w_lo = 0; w_lo < 2; ++w_lo) pack_stage_f16(pk, w->igloo[s].w_v, w_lo, kh, std::ldexp(1.f, e));
      if (dev_upload(h, &h->wpack[2 + s], pk.data(), pk.size())) return 1;
    }
    if (dev_upload(h, &h->conv_bias[0], w->conv2_bias, kC)) return 1;
    if (dev_upload(h, &h->conv_bias[1], w->conv3_bias, kC)) return 1;
  }
  // ---- IGLOO weights
  for (int s = 0; s < 2; ++s) {
    const gnm_igloo_weights& g = w->igloo[s];
    PatchPack pk;
    if (!pack_patches(g.patches, g.w_mult, g.w_summer, pk))
      return fail("gnm_create: IGLOO layer " + std::to_string(s) +
                  ": folded patch weights w_mult * w_summer / 32 not finite: no fp16 operand split carries them");
    h->gather_unscale[s] = pk.unscale;
    h->band_groups[s].resize(kNumBands);
    for (int b = 0; b < kNumBands; ++b) h->band_groups[s][b] = pk.band_gstart[b + 1] - pk.band_gstart[b];
    if (dev_upload(h, &h->grp[s], pk.groups.data(), pk.groups.size())) return 1;
    if (dev_upload(h, &h->band_gstart[s], pk.band_gstart.data(), pk.band_gstart.size())) return 1;
    if (dev_upload(h, reinterpret_cast<uint32_t**>(&h->wfrag[s]), pk.frag.data(), pk.frag.size())) return 1;
    const std::vector<float>& ent_w = pk.ent_w;
    const std::vector<int32_t>&ent_pos = pk.ent_pos, &slot_of = pk.slot_of;
    if (dev_upload(h, &h->ent_w[s], ent_w.data(), ent_w.size())) return 1;
    if (dev_upload(h, &h->ent_pos[s], ent_pos.data(), ent_pos.size())) return 1;
    if (dev_upload(h, &h->slot_of[s], slot_of.data(), slot_of.size())) return 1;
    if (dev_upload(h, &h->wbias[s], g.w_bias, kPatches)) return 1;
    if (dev_upload(h, &h->wqk[s], g.w_qk, static_cast<size_t>(kPatches) * kPooled)) return 1;
    {   // w_qk^T [749][2100] as two TF32 halves: the K-major B operand of logits_tc_kernel
      std::vector<float> thi(static_cast<size_t>(kPooled) * kPatches), tlo(thi.size());
      for (int k = 0; k < kPatches; ++k)
        for (int n = 0; n < kPooled; ++n)
          split_tf32(g.w_qk[static_cast<size_t>(k) * kPooled + n], thi[static_cast<size_t>(n) * kPatches + k],
                     tlo[static_cast<size_t>(n) * kPatches + k]);
      if (dev_upload(h, &h->wqkT_hi[s], thi.data(), thi.size())) return 1;
      if (dev_upload(h, &h->wqkT_lo[s], tlo.data(), tlo.size())) return 1;
    }
    if (dev_upload(h, &h->wv32[s], g.w_v, static_cast<size_t>(kC) * kC)) return 1;
  }
  // ---- head: keras BN inference form  x * inv + (beta - mean * inv),  inv = gamma * rsqrt(var + eps)
  {
    auto bn = [&](const gnm_bn_weights& b, float** scale, float** shift) -> int {
      std::vector<float> sc, sh;
      fold_bn(b, sc, sh);
      if (dev_upload(h, scale, sc.data(), kHidden)) return 1;
      return dev_upload(h, shift, sh.data(), kHidden);
    };
    if (dev_upload(h, &h->d0w, w->dense0_kernel, static_cast<size_t>(256) * kHidden)) return 1;
    if (dev_upload(h, &h->d0b, w->dense0_bias, kHidden)) return 1;
    if (bn(w->bn0, &h->bn0_scale, &h->bn0_shift)) return 1;
    if (dev_upload(h, &h->d1w, w->dense1_kernel, static_cast<size_t>(kHidden) * kHidden)) return 1;
    if (dev_upload(h, &h->d1b, w->dense1_bias, kHidden)) return 1;
    if (bn(w->bn1, &h->bn1_scale, &h->bn1_shift)) return 1;
    const float* dw[2] = {w->dense0_kernel, w->dense1_kernel};
    const int dk[2] = {256, kHidden};
    for (int L = 0; L < 2; ++L) {                          // W^T [512 out][K in] as two TF32 halves: the K-major B operand
      std::vector<float> thi, tlo;
      split_dense_t(dw[L], dk[L], thi, tlo);
      if (dev_upload(h, &h->dwT_hi[L], thi.data(), thi.size())) return 1;
      if (dev_upload(h, &h->dwT_lo[L], tlo.data(), tlo.size())) return 1;
    }
    if (dev_upload(h, &h->d2w, w->dense2_kernel, static_cast<size_t>(kHidden) * 3)) return 1;
    if (dev_upload(h, &h->d2b, w->dense2_bias, 3)) return 1;
  }
  // ---- workspace
  const size_t mb = static_cast<size_t>(max_batch);
  h->mb_pad = (max_batch + kBandWins - 1) / kBandWins * kBandWins;
  const size_t mbp = static_cast<size_t>(h->mb_pad);
  for (int i = 0; i < 2; ++i) {
    if (dev_alloc(h, &h->ybuf[i], mbp * kTok * kRowBytes)) return 1;      // whole window groups: wv_gather_kernel reads n_pad windows
    for (int par = 0; par < 2; ++par) {
      if (dev_alloc(h, &h->q_set[par][i], mb * kPooled * kC)) return 1;
      if (dev_alloc(h, &h->mpi_set[par][i], mb * kPatches)) return 1;
      if (dev_alloc(h, &h->mpi_hi_set[par][i], mb * kPatches)) return 1;
      if (dev_alloc(h, &h->mpi_lo_set[par][i], mb * kPatches)) return 1;
    }
    h->q[i] = h->q_set[0][i]; h->mpi[i] = h->mpi_set[0][i]; h->mpi_hi[i] = h->mpi_hi_set[0][i]; h->mpi_lo[i] = h->mpi_lo_set[0][i];
    if (dev_alloc(h, &h->in_stage[i], mb * kWindow)) return 1;
    if (dev_alloc(h, &h->out_stage[i], mb * 3)) return 1;
    GNM_CUDA(cudaEventCreateWithFlags(&h->in_ready[i], cudaEventDisableTiming));
    GNM_CUDA(cudaEventCreateWithFlags(&h->in_free[i], cudaEventDisableTiming));
  }
  if (dev_alloc(h, &h->conv_dbg, static_cast<size_t>(h->num_sms) * 8)) return 1;
  GNM_CUDA(cudaMemset(h->conv_dbg, 0, static_cast<size_t>(h->num_sms) * 8 * sizeof(long long)));
  if (dev_alloc(h, &h->part, mbp * kGsSlots)) return 1;
  if (dev_alloc(h, &h->cta_split, static_cast<size_t>(2) * (h->num_sms + 1))) return 1;
  if (dev_alloc(h, &h->logits, mb * kLogitsLd)) return 1;
  if (dev_alloc(h, &h->logits_part, mb * kLogitsLd * kLgSplits)) return 1;
  if (dev_alloc(h, &h->h0, mb * 256)) return 1;
  if (dev_alloc(h, &h->h1, mb * kHidden)) return 1;
  if (dev_alloc(h, &h->h2, mb * kHidden)) return 1;
  if (dev_alloc(h, &h->hA_hi[0], mb * 256)) return 1;
  if (dev_alloc(h, &h->hA_lo[0], mb * 256)) return 1;
  if (dev_alloc(h, &h->hA_hi[1], mb * kHidden)) return 1;
  if (dev_alloc(h, &h->hA_lo[1], mb * kHidden)) return 1;
  GNM_CUDA(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
  GNM_CUDA(cudaStreamCreateWithFlags(&h->compute_stream, cudaStreamNonBlocking));
  {
    int prio_lo = 0, prio_hi = 0;
    GNM_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    GNM_CUDA(cudaStreamCreateWithPriority(&h->tail_stream, cudaStreamNonBlocking, prio_hi));   // few small CTAs: schedule them promptly
    for (int i = 0; i < 2; ++i) {
      GNM_CUDA(cudaEventCreateWithFlags(&h->main_done[i], cudaEventDisableTiming));
      GNM_CUDA(cudaEventCreateWithFlags(&h->tail_done[i], cudaEventDisableTiming));
    }
  }
  GNM_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&h->status), sizeof(DeviceStatus), cudaHostAllocMapped));
  std::memset(h->status, 0, sizeof(DeviceStatus));

  // ---- TMA descriptors
  PFN_encodeTiled enc = nullptr;
  if (get_encode_fn(&enc)) return 1;
  for (int i = 0; i < 2; ++i) {
    if (make_act_map(enc, &h->tm_act[i], h->ybuf[i], max_batch)) return 1;
    if (make_band_map(enc, &h->tm_band[i], h->ybuf[i], h->mb_pad)) return 1;
  }
  for (int i = 0; i < 4; ++i) {
    const int n_stages = i < 2 ? kConvStages : kWvStages;
    if (make_w_map(enc, &h->tm_w[i], h->wpack[i], n_stages, 128)) return 1;
    if (make_w_map(enc, &h->tm_w_half[i], h->wpack[i], n_stages, 64)) return 1;
  }
  for (int s = 0; s < 2; ++s) {
    for (int par = 0; par < 2; ++par) {
      if (make_f32_map(enc, &h->tm_lg_a_set[par][s][0], h->mpi_hi_set[par][s], kPatches, max_batch, kLgBM)) return 1;
      if (make_f32_map(enc, &h->tm_lg_a_set[par][s][1], h->mpi_lo_set[par][s], kPatches, max_batch, kLgBM)) return 1;
    }
    h->tm_lg_a[s][0] = h->tm_lg_a_set[0][s][0]; h->tm_lg_a[s][1] = h->tm_lg_a_set[0][s][1];
    if (make_f32_map(enc, &h->tm_lg_b[s][0], h->wqkT_hi[s], kPatches, kPooled, kLgBN)) return 1;
    if (make_f32_map(enc, &h->tm_lg_b[s][1], h->wqkT_lo[s], kPatches, kPooled, kLgBN)) return 1;
  }

  for (int L = 0; L < 2; ++L) {
    const int K = L == 0 ? 256 : kHidden;
    if (make_f32_map(enc, &h->tm_hd_a[L][0], h->hA_hi[L], K, max_batch, kLgBM)) return 1;
    if (make_f32_map(enc, &h->tm_hd_a[L][1], h->hA_lo[L], K, max_batch, kLgBM)) return 1;
    if (make_f32_map(enc, &h->tm_hd_b[L][0], h->dwT_hi[L], K, kHidden, kLgBN)) return 1;
    if (make_f32_map(enc, &h->tm_hd_b[L][1], h->dwT_lo[L], K, kHidden, kLgBN)) return 1;
  }

  // ---- opt in to large dynamic shared memory
  GNM_CUDA(cudaFuncSetAttribute(conv_t_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvTSmem));
  GNM_CUDA(cudaFuncSetAttribute(conv_t_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvTSmem));
  GNM_CUDA(cudaFuncSetAttribute(wv_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem));
  GNM_CUDA(cudaFuncSetAttribute(layer1_wv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFuSmem));
  GNM_CUDA(cudaFuncSetAttribute(layer1_wv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFuSmem));
  GNM_CUDA(cudaFuncSetAttribute(logits_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLgSmem));
  GNM_CUDA(cudaFuncSetAttribute(conv_ref_kernel<6, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ref_smem_bytes<6>()));
  GNM_CUDA(cudaFuncSetAttribute(conv_ref_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ref_smem_bytes<1>()));
  GNM_CUDA(cudaDeviceSynchronize());
  return 0;
}

extern "C" int gnm_destroy(gnm_handle* h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  for (void* p : h->allocs) cudaFree(p);
  if (h->scratch32) cudaFree(h->scratch32);
  for (int i = 0; i < 2; ++i) {
    if (h->in_ready[i]) cudaEventDestroy(h->in_ready[i]);
    if (h->in_free[i]) cudaEventDestroy(h->in_free[i]);
  }
  for (cudaEvent_t e : h->timer.events) cudaEventDestroy(e);
  for (int i = 0; i < 2; ++i) {
    if (h->main_done[i]) cudaEventDestroy(h->main_done[i]);
    if (h->tail_done[i]) cudaEventDestroy(h->tail_done[i]);
  }
  if (h->tail_stream) cudaStreamDestroy(h->tail_stream);
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  if (h->compute_stream) cudaStreamDestroy(h->compute_stream);
  if (h->status) cudaFreeHost(h->status);
  delete h;
  return 0;
}

// ------------------------------------------------------------------------------------------------
template <class O>
static int check_launch(O* h, const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(std::string(what) + " launch failed: " + cudaGetErrorString(e));
  h->launches++;
  return 0;
}

static void timer_mark(gnm_handle* h, const char* name, cudaStream_t st) {
  if (!h->profile_stages) return;
  StageTimer& t = h->timer;
  const size_t i = t.names.size();
  if (t.events.size() <= i) { cudaEvent_t e; cudaEventCreate(&e); t.events.push_back(e); }
  cudaEventRecord(t.events[i], st);
  t.names.push_back(name);
}

// layer 0: conv2 (y[in] -> y[1-in], planes hi16 + lo8 + hi8 for conv3); layer 1: conv3 (planes hi16 + lo16)
static int launch_conv(gnm_handle* h, int layer, int in_buf, int n, cudaStream_t st) {
  ConvTcParams p;
  p.n_tiles = n * kUnitsPerWin;                  // 256-position units
  p.status = h->status;
  p.experiment = h->conv_experiment;
  // bit 4: cycle counters of conv3 (layer 1); bit 8: of conv2 (layer 0)
  p.dbg = ((h->conv_experiment & 4) && layer == 1) || ((h->conv_experiment & 8) && layer == 0) ? h->conv_dbg : nullptr;
  p.bias = h->conv_bias[layer];
  p.y_out = h->ybuf[1 - in_buf];
  p.q_out = nullptr;
  p.out_scale = h->conv_out_scale[layer];
  p.out_fp8 = layer == 0 ? 1 : 0;
  h->ybuf_fp8lo[1 - in_buf] = p.out_fp8;
  int grid = std::min(h->num_sms, p.n_tiles);
  if (h->conv_cluster > 1 && grid >= h->conv_cluster) {
    // Experiment: launch the persistent CTAs as thread-block clusters.  Nothing in the kernel changes (every CTA still issues
    // its own unicast TMA loads); the question is whether L2 deduplicates the identical weight-stage requests of a cluster's
    // CTAs.  The grid must be a whole number of co-resident clusters.
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = h->conv_cluster; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.blockDim = dim3(kConvThreads); cfg.dynamicSmemBytes = kConvTSmem; cfg.stream = st; cfg.attrs = attr; cfg.numAttrs = 1;
    cfg.gridDim = dim3(grid / h->conv_cluster * h->conv_cluster);
    int max_clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&max_clusters, conv_t_kernel<false>, &cfg) == cudaSuccess && max_clusters > 0)
      grid = std::min(grid / h->conv_cluster, max_clusters) * h->conv_cluster;
    else
      grid = grid / h->conv_cluster * h->conv_cluster;
    cfg.gridDim = dim3(grid);
    GNM_CUDA(cudaLaunchKernelEx(&cfg, conv_t_kernel<false>, h->tm_act[in_buf], h->tm_w_half[layer], p));
    return check_launch(h, "conv_t_kernel<false>(cluster)");
  }
  conv_t_kernel<false><<<grid, kConvThreads, kConvTSmem, st>>>(h->tm_act[in_buf], h->tm_w_half[layer], p);
  return check_launch(h, "conv_t_kernel<false>");
}
// q[s] = maxpool8(y[buf] @ w_v#s)
static int launch_wv_tc(gnm_handle* h, int s, int buf, int n, cudaStream_t st) {
  ConvTcParams p;
  p.status = h->status;
  p.experiment = 0;
  p.dbg = nullptr;
  p.bias = nullptr; p.y_out = nullptr; p.q_out = h->q[s];
  p.out_scale = h->wv_out_scale[s];
  p.out_fp8 = 0;
  p.n_tiles = n * kUnitsPerWin;
  const int grid = std::min(h->num_sms, p.n_tiles);
  conv_t_kernel<true><<<grid, kConvThreads, kConvTSmem, st>>>(h->tm_act[buf], h->tm_w_half[2 + s], p);
  return check_launch(h, "conv_t_kernel<true>");
}

// Unit ranges of wv_gather_kernel's CTAs.  A unit's cost is ~ (streaming its 128 KB of activations) + (its band's entries x 8
// windows of gather arithmetic); bands hold 45 +- 7 entries (more in adversarial patch sets), so an equal-count split leaves
// the CTAs that own entry-rich bands as stragglers.  Cost model: a unit costs wv_cost_base plus wv_cost_group per position group
// of its band's busiest gather warp.  Recomputed only when the window-group count or the grid changes; uploaded on the caller's stream.
static int wv_split(gnm_handle* h, int s, int groups, int grid, cudaStream_t st) {
  if (h->split_groups[s] == groups && h->split_grid[s] == grid) return 0;
  std::vector<double> cost(kNumBands);
  double total = 0;
  for (int b = 0; b < kNumBands; ++b) {
    const int per_warp = (h->band_groups[s][b] + kWgWarps - 1) / kWgWarps;
    cost[b] = h->wv_cost_base + h->wv_cost_group * per_warp;
    total += cost[b] * groups;
  }
  std::vector<int32_t>& sp = h->split_host[s];
  sp.assign(h->num_sms + 1, kNumBands * groups);
  sp[0] = 0;
  double acc = 0;
  int c = 1;
  for (int b = 0; b < kNumBands && c < grid; ++b)
    for (int g = 0; g < groups && c < grid; ++g) {
      acc += cost[b];
      if (acc >= total * c / grid) sp[c++] = b * groups + g + 1;
    }
  for (; c <= grid; ++c) sp[c] = kNumBands * groups;
  for (int i = 1; i <= grid; ++i) sp[i] = std::max(sp[i], sp[i - 1]);
  GNM_CUDA(cudaMemcpyAsync(h->cta_split + s * (h->num_sms + 1), sp.data(), (grid + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  h->split_groups[s] = groups; h->split_grid[s] = grid;
  return 0;
}

// IGLOO kernel s on y[buf]: q[s] = maxpool8(y @ w_v#s) and mpi[s] (patch gather) in ONE pass over the activations
static int launch_wv_gather(gnm_handle* h, int s, int buf, int n, cudaStream_t st) {
  WvGatherParams p;
  p.q_out = h->q[s]; p.out_scale = h->wv_out_scale[s];
  p.grp = h->grp[s]; p.band_gstart = h->band_gstart[s]; p.wfrag = h->wfrag[s]; p.gather_unscale = h->gather_unscale[s]; p.part_t = h->part;
  p.n_windows = n;
  p.n_pad = (n + kBandWins - 1) / kBandWins * kBandWins;
  p.groups = p.n_pad / kBandWins;
  p.n_units = kNumBands * p.groups;
  p.status = h->status;
  p.experiment = h->conv_experiment;
  p.dbg = (h->conv_experiment & 512) && s == 1 ? h->conv_dbg : nullptr;      // cycle counters of the IGLOO#1 launch
  const int grid = std::min(h->num_sms, p.n_units);
  if (wv_split(h, s, p.groups, grid, st)) return 1;
  p.cta_split = h->cta_split + s * (h->num_sms + 1);
  wv_gather_kernel<<<grid, kWgThreads, kWgSmem, st>>>(h->tm_band[buf], h->tm_w[2 + s], p);
  if (check_launch(h, "wv_gather_kernel")) return 1;
  dim3 fgrid((kPatches + 31) / 32, (n + 31) / 32);
  patch_finish_t_kernel<<<fgrid, 256, 0, st>>>(h->part, h->slot_of[s], h->wbias[s], h->mpi[s], h->mpi_hi[s], h->mpi_lo[s], n, p.n_pad);
  return check_launch(h, "patch_finish_t_kernel");
}

static int ensure_scratch(gnm_handle* h) {
  if (h->scratch32) return 0;
  GNM_CUDA(cudaMalloc(reinterpret_cast<void**>(&h->scratch32), static_cast<size_t>(h->max_batch) * kTok * kC * sizeof(float)));
  return 0;
}

static int launch_conv_ref(gnm_handle* h, int layer, int in_buf, int n, cudaStream_t st) {
  if (ensure_scratch(h)) return 1;
  dim3 grid((kTok + kRefPos - 1) / kRefPos, n);
  conv_ref_kernel<6, true><<<grid, kRefThreads, ref_smem_bytes<6>(), st>>>(h->ybuf[in_buf], h->conv_w32[layer],
                                                                          h->conv_bias[layer], h->scratch32);
  if (check_launch(h, "conv_ref_kernel")) return 1;
  const size_t rows = static_cast<size_t>(n) * kTok;
  const size_t threads = rows * (kC / 4);
  split_rows_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, st>>>(h->scratch32, h->ybuf[1 - in_buf], rows);
  return check_launch(h, "split_rows_kernel");
}
static int launch_wv_ref(gnm_handle* h, int s, int in_buf, int n, cudaStream_t st) {
  if (ensure_scratch(h)) return 1;
  dim3 grid((kTok + kRefPos - 1) / kRefPos, n);
  conv_ref_kernel<1, false><<<grid, kRefThreads, ref_smem_bytes<1>(), st>>>(h->ybuf[in_buf], h->wv32[s], nullptr, h->scratch32);
  if (check_launch(h, "conv_ref_kernel<1>")) return 1;
  const size_t total = static_cast<size_t>(n) * kPooled * kC;
  maxpool8_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(h->scratch32, h->q[s], n);
  return check_launch(h, "maxpool8_kernel");
}

static int launch_gather(gnm_handle* h, int s, int buf, int n, cudaStream_t st) {
  patch_stream_kernel<<<kGsGroups, kGsThreads, 0, st>>>(h->ybuf[buf], h->ent_pos[s], h->ent_w[s], h->part, n);
  if (check_launch(h, "patch_stream_kernel")) return 1;
  dim3 grid((kPatches + 255) / 256, n);
  patch_finish_kernel<<<grid, 256, 0, st>>>(h->part, h->slot_of[s], h->wbias[s], h->mpi[s], h->mpi_hi[s], h->mpi_lo[s], n);
  return check_launch(h, "patch_finish_kernel");
}

template <class O>     // O: the handle, or a head trainer (anything that counts its launches)
static int launch_sgemm(O* h, const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N,
                        int K, const float* bias, const float* scale, const float* shift, int relu, cudaStream_t st) {
  const int nb = (N + kGemmBN - 1) / kGemmBN;
  if (M >= 64) {                                           // 32-row tiles only for tiny batches (measured slower otherwise)
    dim3 grid(nb, (M + 63) / 64);
    sgemm_epi_kernel<64><<<grid, 256, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K, bias, scale, shift, relu, K);
  } else {
    dim3 grid(nb, (M + 31) / 32);
    sgemm_epi_kernel<32><<<grid, 128, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K, bias, scale, shift, relu, K);
  }
  return check_launch(h, "sgemm_epi_kernel");
}

// logits = mpi @ w_qk: M = n windows is small (192 tiles of 64x64 at batch 1024), so K = 2100 is split 4 ways to put
// ~5 CTAs on every SM; the partials are summed in fixed order by splitk_reduce_kernel.
constexpr int kLogitsSplit = 4;
static int launch_logits(gnm_handle* h, int s, int n, cudaStream_t st) {
  int parts;
  if (h->conv_impl == 0) {
    // tensor cores, 3 x TF32 (logits_tc.cuh): 3 N tiles x ceil(n/128) M tiles x 6 K splits
    LogitsTcParams p;
    p.part = h->logits_part; p.ldc = kLogitsLd; p.n_rows = n; p.n_cols = kPooled; p.status = h->status;
    p.chunks_total = kLgChunks; p.chunks_per_split = kLgChunksPerSplit;
    dim3 grid((kPooled + kLgBN - 1) / kLgBN, (n + kLgBM - 1) / kLgBM, kLgSplits);
    logits_tc_kernel<<<grid, kLgThreads, kLgSmem, st>>>(h->tm_lg_a[s][0], h->tm_lg_a[s][1], h->tm_lg_b[s][0], h->tm_lg_b[s][1], p);
    if (check_launch(h, "logits_tc_kernel")) return 1;
    parts = kLgSplits;
  } else {
    // fp32 FFMA validation path (conv_impl = 1): 64x64 tiles, K split 4 ways
    const int k_chunk = ((kPatches + kLogitsSplit - 1) / kLogitsSplit + kGemmBK - 1) / kGemmBK * kGemmBK;   // 528
    dim3 grid((kPooled + kGemmBN - 1) / kGemmBN, (n + 63) / 64, kLogitsSplit);
    sgemm_epi_kernel<64><<<grid, 256, 0, st>>>(h->mpi[s], kPatches, h->wqk[s], kPooled, h->logits_part, kLogitsLd, n, kPooled,
                                              kPatches, nullptr, nullptr, nullptr, 0, k_chunk);
    if (check_launch(h, "sgemm_epi_kernel(split-K)")) return 1;
    parts = kLogitsSplit;
  }
  const size_t total = static_cast<size_t>(n) * kLogitsLd;
  splitk_reduce_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(h->logits_part, h->logits, n, kLogitsLd,
                                                                                    kPooled, parts);
  return check_launch(h, "splitk_reduce_kernel");
}

// Dense(512) + BatchNorm + ReLU of the head on the tensor cores: out = relu(bn(A @ W + b)), A given as TF32 halves (layer 0: h0
// [n][256] written by attention_kernel, layer 1: h1 [n][512] written by the previous call), 3 x TF32 passes, K split 8 ways so
// 128 CTAs run at batch 1024; the split-K partials go through logits_part (6 x 752 floats per window >= 8 x 512).
constexpr int kHeadSplits = 8;
static_assert(kHeadSplits * kHidden <= kLgSplits * kLogitsLd, "logits_part is too small for the head's split-K partials");
static int launch_dense_tc_maps(gnm_handle* h, const CUtensorMap* tm_a, const CUtensorMap* tm_b, int K, int n, const float* bias,
                                const float* scale, const float* shift, float* out, float* out_hi, float* out_lo, float* emit,
                                cudaStream_t st) {
  LogitsTcParams p;
  p.part = h->logits_part; p.ldc = kHidden; p.n_rows = n; p.n_cols = kHidden; p.status = h->status;
  p.chunks_total = K / kLgBK;
  p.chunks_per_split = (p.chunks_total + kHeadSplits - 1) / kHeadSplits;
  const int splits = (p.chunks_total + p.chunks_per_split - 1) / p.chunks_per_split;
  dim3 grid(kHidden / kLgBN, (n + kLgBM - 1) / kLgBM, splits);
  logits_tc_kernel<<<grid, kLgThreads, kLgSmem, st>>>(tm_a[0], tm_a[1], tm_b[0], tm_b[1], p);
  if (check_launch(h, "logits_tc_kernel(dense)")) return 1;
  const size_t total = static_cast<size_t>(n) * kHidden;
  splitk_reduce_epi_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
      h->logits_part, out, out_hi, out_lo, emit, n, kHidden, splits, bias, scale, shift, 1);
  return check_launch(h, "splitk_reduce_epi_kernel");
}
static int launch_dense_tc(gnm_handle* h, int layer, int n, float* out, float* out_hi, float* out_lo, float* emit, cudaStream_t st) {
  return launch_dense_tc_maps(h, h->tm_hd_a[layer], h->tm_hd_b[layer], layer == 0 ? 256 : kHidden, n, layer == 0 ? h->d0b : h->d1b,
                              layer == 0 ? h->bn0_scale : h->bn1_scale, layer == 0 ? h->bn0_shift : h->bn1_shift, out, out_hi,
                              out_lo, emit, st);
}

// the buffer set the next step's main part writes and its tail reads (kernel arguments are captured at launch, so switching the
// "current" pointers between steps is all it takes)
static void select_set(gnm_handle* h, int par) {
  for (int s = 0; s < 2; ++s) {
    h->q[s] = h->q_set[par][s]; h->mpi[s] = h->mpi_set[par][s];
    h->mpi_hi[s] = h->mpi_hi_set[par][s]; h->mpi_lo[s] = h->mpi_lo_set[par][s];
    h->tm_lg_a[s][0] = h->tm_lg_a_set[par][s][0]; h->tm_lg_a[s][1] = h->tm_lg_a_set[par][s][1];
  }
}

// Layer 1 of an integrated-gradients step (encode.cuh, embed_conv1_ig_kernel): row r is window r / m of d_ascii at
// alpha = (r mod m + 1/2) / m on the line from the baseline (kIgZero / kIgN) to the window; m = 0: the baseline itself.
struct L1Interp {
  int m, baseline;
};

// main part of a step: layer 1, the two IGLOO kernels' value projection + patch gather, conv2, conv3 (everything that streams
// the activations); returns 2 when a debug_stop cut the step short.  With `ig`, layer 1 is the interpolated embed kernel
// whatever fuse_l1 says (ASCII input only), and the rest of the step is unchanged.
static int forward_main(gnm_handle* h, const uint8_t* d_ascii, const uint16_t* d_tok, int n, cudaStream_t st,
                        const L1Interp* ig = nullptr) {
  dim3 egrid((kTok + kEmbSeg - 1) / kEmbSeg, n);
  h->ybuf_fp8lo[0] = h->ybuf_fp8lo[1] = 0;
  const bool fused = h->fuse_l1 && h->conv_impl == 0 && !ig;       // layer 1 + w_v#0 in one kernel
  if (ig) {
    timer_mark(h, "embed_conv1_ig", st);
    embed_conv1_ig_kernel<<<egrid, kEmbThreads, 0, st>>>(d_ascii, h->conv1_table, h->conv1_triple, h->conv1_bias, h->ybuf[0],
                                                         ig->m, ig->baseline, h->status);
    if (check_launch(h, "embed_conv1_ig_kernel")) return 1;
  } else if (fused) {
    timer_mark(h, "layer1_wv0", st);
    FusedParams fp;
    fp.ascii = d_ascii; fp.tokens = d_tok; fp.table = h->conv1_table; fp.triple = h->conv1_triple; fp.bias = h->conv1_bias;
    fp.y_out = h->ybuf[0]; fp.q_out = h->q[0]; fp.q_scale = h->wv_out_scale[0]; fp.n_units = n * kFuUnitsPerWin; fp.status = h->status;
    const int grid = std::min(h->num_sms, fp.n_units);
    if (d_ascii) layer1_wv_kernel<true><<<grid, kFuThreads, kFuSmem, st>>>(h->tm_w[2], fp);
    else layer1_wv_kernel<false><<<grid, kFuThreads, kFuSmem, st>>>(h->tm_w[2], fp);
    if (check_launch(h, "layer1_wv_kernel")) return 1;
  } else {
  timer_mark(h, "embed_conv1", st);
  if (d_ascii)
    embed_conv1_kernel<true><<<egrid, kEmbThreads, 0, st>>>(d_ascii, nullptr, h->conv1_table, h->conv1_triple, h->conv1_bias, h->ybuf[0], n, h->status);
  else
    embed_conv1_kernel<false><<<egrid, kEmbThreads, 0, st>>>(nullptr, d_tok, h->conv1_table, h->conv1_triple, h->conv1_bias, h->ybuf[0], n, h->status);
  if (check_launch(h, "embed_conv1_kernel")) return 1;
  }
  const bool fg = h->fuse_gather && h->conv_impl == 0 && !fused;     // w_v + gather in one kernel (wv_gather.cuh)
  if (fg) {
    timer_mark(h, "wvg0", st);
    if (launch_wv_gather(h, 0, 0, n, st)) return 1;          // y1 (buf0) -> q0, mpi0
  } else {
    timer_mark(h, "gather0", st);
    if (launch_gather(h, 0, 0, n, st)) return 1;
  }
  if (h->debug_stop == 1) { timer_mark(h, "end", st); return 2; }
  if (h->conv_impl == 0) {
    if (!fused && !fg) {
      timer_mark(h, "wv0", st);
      if (launch_wv_tc(h, 0, 0, n, st)) return 1;             // y1 (buf0) -> q0
    }
    timer_mark(h, "conv2", st);
    if (launch_conv(h, 0, 0, n, st)) return 1;             // y1 (buf0) -> y2 (buf1)
    if (h->debug_stop == 2) { timer_mark(h, "end", st); return 2; }
    timer_mark(h, "conv3", st);
    if (launch_conv(h, 1, 1, n, st)) return 1;             // y2 (buf1) -> y3 (buf0)
    if (h->debug_stop == 3) { timer_mark(h, "end", st); return 2; }
    if (fg) {
      timer_mark(h, "wvg1", st);
      if (launch_wv_gather(h, 1, 0, n, st)) return 1;        // y3 (buf0) -> q1, mpi1
    } else {
      timer_mark(h, "wv1", st);
      if (launch_wv_tc(h, 1, 0, n, st)) return 1;               // y3 (buf0) -> q1
    }
  } else {
    timer_mark(h, "wv0(ref)", st);
    if (launch_wv_ref(h, 0, 0, n, st)) return 1;
    timer_mark(h, "conv2(ref)", st);
    if (launch_conv_ref(h, 0, 0, n, st)) return 1;
    if (h->debug_stop == 2) { timer_mark(h, "end", st); return 2; }
    timer_mark(h, "conv3(ref)", st);
    if (launch_conv_ref(h, 1, 1, n, st)) return 1;
    if (h->debug_stop == 3) { timer_mark(h, "end", st); return 2; }
    timer_mark(h, "wv1(ref)", st);
    if (launch_wv_ref(h, 1, 0, n, st)) return 1;
  }
  if (!fg) {
    timer_mark(h, "gather1", st);
    if (launch_gather(h, 1, 0, n, st)) return 1;
  }
  return 0;
}

// tail of a step: attention logits, softmax + weighted sum, dense head -> probabilities.  Small kernels
// that read only q / mpi of the current buffer set and the tail-only buffers (logits, h0..h2).
// d_embed (the step's first row, or null): dense layer 0's output h1 -- the encoder's output -- is also stored there; with
// d_probs null the head stops after that layer.
static int forward_tail(gnm_handle* h, int n, float* d_probs, float* d_embed, cudaStream_t st) {
  for (int s = 0; s < 2; ++s) {
    timer_mark(h, s ? "logits1" : "logits0", st);
    if (launch_logits(h, s, n, st)) return 1;
    timer_mark(h, s ? "attention1" : "attention0", st);
    attention_kernel<<<n, 128, 0, st>>>(h->logits, h->q[s], h->h0, h->hA_hi[0], h->hA_lo[0], s * kC);
    if (check_launch(h, "attention_kernel")) return 1;
  }
  timer_mark(h, "head", st);
  if (h->conv_impl == 0) {       // tensor cores, 3 x TF32 (the model's dense projections; the FFMA kernels stay the validation path)
    if (launch_dense_tc(h, 0, n, h->h1, h->hA_hi[1], h->hA_lo[1], d_embed, st)) return 1;
    if (!d_probs) { timer_mark(h, "end", st); return 0; }
    if (launch_dense_tc(h, 1, n, h->h2, nullptr, nullptr, nullptr, st)) return 1;
  } else {
    if (launch_sgemm(h, h->h0, 256, h->d0w, kHidden, h->h1, kHidden, n, kHidden, 256, h->d0b, h->bn0_scale, h->bn0_shift, 1, st)) return 1;
    if (d_embed)
      GNM_CUDA(cudaMemcpyAsync(d_embed, h->h1, static_cast<size_t>(n) * kHidden * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (!d_probs) { timer_mark(h, "end", st); return 0; }
    if (launch_sgemm(h, h->h1, kHidden, h->d1w, kHidden, h->h2, kHidden, n, kHidden, kHidden, h->d1b, h->bn1_scale, h->bn1_shift, 1, st)) return 1;
  }
  dense3_softmax_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(h->h2, h->d2w, h->d2b, d_probs, n);
  if (check_launch(h, "dense3_softmax_kernel")) return 1;
  timer_mark(h, "end", st);
  return 0;
}

// One step: n <= max_batch windows (or interpolated rows, see forward_main), strictly in order on one stream.
static int forward_step(gnm_handle* h, const uint8_t* d_ascii, const uint16_t* d_tok, int n, float* d_probs, float* d_embed,
                        cudaStream_t st, const L1Interp* ig = nullptr) {
  const int rc = forward_main(h, d_ascii, d_tok, n, st, ig);
  if (rc) return rc == 2 ? 0 : 1;
  return forward_tail(h, n, d_probs, d_embed, st);
}

// Steps of a multi-step call with the tails overlapped: the main part of step i+1 (which starts with the issue-bound layer-1
// kernel, small CTAs, no dynamic shared memory) runs on `st` while the few small kernels of step i's tail run on the
// high-priority tail_stream next to it.  Two buffer sets alternate; main(i) waits for tail(i-2) (same set), tail(i) waits for
// main(i); `st` is joined with both tails before the call returns, so the caller's stream semantics are unchanged.
struct TailOverlap {
  gnm_handle* h; cudaStream_t st; int steps_done = 0;
  bool on;
  TailOverlap(gnm_handle* h_, cudaStream_t st_, int n_steps)
      : h(h_), st(st_), on(h_->tail_overlap && n_steps > 1 && !h_->profile_stages && h_->debug_stop == 0) {}
  int step(const uint8_t* d_ascii, const uint16_t* d_tok, int n, float* d_probs, float* d_embed, cudaStream_t* tail_out = nullptr) {
    if (tail_out) *tail_out = st;
    if (!on) return forward_step(h, d_ascii, d_tok, n, d_probs, d_embed, st);
    const int par = steps_done & 1;
    select_set(h, par);
    if (steps_done >= 2) GNM_CUDA(cudaStreamWaitEvent(st, h->tail_done[par], 0));
    const int rc = forward_main(h, d_ascii, d_tok, n, st);
    if (rc) return 1;
    GNM_CUDA(cudaEventRecord(h->main_done[par], st));
    GNM_CUDA(cudaStreamWaitEvent(h->tail_stream, h->main_done[par], 0));
    if (forward_tail(h, n, d_probs, d_embed, h->tail_stream)) return 1;
    if (tail_out) *tail_out = h->tail_stream;
    GNM_CUDA(cudaEventRecord(h->tail_done[par], h->tail_stream));
    ++steps_done;
    return 0;
  }
  int join() {                                           // `st` continues only after every tail has finished
    if (!on) return 0;
    for (int k = 0; k < 2 && k < steps_done; ++k) GNM_CUDA(cudaStreamWaitEvent(st, h->tail_done[(steps_done - 1 - k) & 1], 0));
    select_set(h, (steps_done - 1) & 1);                 // debug_fetch sees the last step's buffers
    return 0;
  }
};

static int check_device_status(gnm_handle* h) {
  if (h->status && h->status->act_overflow) {
    // not fatal for the device, but the parity promise no longer holds for the step that raised it: fail loudly
    const int stage = h->status->ov_stage[1] ? 1 : h->status->ov_stage[2] ? 2 : h->status->ov_stage[3] ? 3 : 0;   // the first layer that left the range
    h->status->act_overflow = 0;
    for (int i = 0; i < 4; ++i) h->status->ov_stage[i] = 0;
    if (stage == 0)
      return fail("gradient range exceeded in the backward pass of an attribution call: a gradient is not finite, or its "
                  "per-window scale cannot bring it under 3.5 -- the attributions of that step are not within their precision bar");
    return fail(std::string("activation range exceeded in ") + (stage == 1 ? "layer 1" : stage == 2 ? "conv2" : "conv3") +
                ": |y| > 3.5 saturates the e4m3 correction plane (|y| > 2047 overflows fp16) -- these weights are outside the "
                "range the split-operand tensor-core recipe supports (common.cuh); results of that step are not within 1e-4");
  }
  if (h->status && h->status->code != kDevOk) {
    char buf[160];
    std::snprintf(buf, sizeof buf, "device-side failure %d (mbarrier timeout) tag=%d block=%d thread=%d",
                  h->status->code, h->status->info0, h->status->info1, h->status->info2);
    return fail(buf);
  }
  return 0;
}

// d_probs + off * 3 / d_embed + off * 512 of the step that starts at window `off` (null stays null)
static float* probs_at(float* d_probs, int off) { return d_probs ? d_probs + static_cast<size_t>(off) * 3 : nullptr; }
static float* embed_at(float* d_embed, int off) { return d_embed ? d_embed + static_cast<size_t>(off) * kHidden : nullptr; }

static int forward_any(gnm_handle* h, const uint8_t* d_ascii, const uint16_t* d_tok, int n, float* d_probs, float* d_embed,
                       void* stream) {
  if (!h) return fail("null handle");
  if (n < 0) return fail("negative window count");
  if (n == 0) return 0;
  if ((!d_ascii && !d_tok) || (!d_probs && !d_embed)) return fail("null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  if (check_device_status(h)) return 1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TailOverlap ov(h, st, (n + h->max_batch - 1) / h->max_batch);
  for (int off = 0; off < n; off += h->max_batch) {
    const int m = std::min(h->max_batch, n - off);
    if (ov.step(d_ascii ? d_ascii + static_cast<size_t>(off) * kWindow : nullptr,
                d_tok ? d_tok + static_cast<size_t>(off) * kTok : nullptr, m, probs_at(d_probs, off), embed_at(d_embed, off))) return 1;
  }
  return ov.join();
}

extern "C" int gnm_forward_ascii(gnm_handle* h, const uint8_t* d_ascii, int n, float* d_probs, void* stream) {
  return forward_any(h, d_ascii, nullptr, n, d_probs, nullptr, stream);
}
extern "C" int gnm_forward_tokens(gnm_handle* h, const uint16_t* d_tokens, int n, float* d_probs, void* stream) {
  return forward_any(h, nullptr, d_tokens, n, d_probs, nullptr, stream);
}
extern "C" int gnm_embed_ascii(gnm_handle* h, const uint8_t* d_ascii, int n, float* d_probs, float* d_embed, void* stream) {
  if (!d_embed && n > 0) return fail("gnm_embed_ascii: d_embed is null");
  return forward_any(h, d_ascii, nullptr, n, d_probs, d_embed, stream);
}
extern "C" int gnm_embed_tokens(gnm_handle* h, const uint16_t* d_tokens, int n, float* d_probs, float* d_embed, void* stream) {
  if (!d_embed && n > 0) return fail("gnm_embed_tokens: d_embed is null");
  return forward_any(h, nullptr, d_tokens, n, d_probs, d_embed, stream);
}

extern "C" int gnm_encode(gnm_handle* h, const uint8_t* d_ascii, int n, uint16_t* d_tokens, void* stream) {
  if (!h) return fail("null handle");
  if (n < 0) return fail("negative window count");
  if (n == 0) return 0;
  if (!d_ascii || !d_tokens) return fail("null buffer");
  if (reinterpret_cast<uintptr_t>(d_ascii) % 16) return fail("gnm_encode: d_ascii must be 16-byte aligned");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int off = 0; off < n; off += 32768) {                     // gridDim.y limit is 65535
    const int m = std::min(32768, n - off);
    dim3 grid((kTok + kEncSeg - 1) / kEncSeg, m);
    encode_tokens_kernel<<<grid, kEncThreads, 0, st>>>(d_ascii + static_cast<size_t>(off) * kWindow,
                                                      d_tokens + static_cast<size_t>(off) * kTok, m);
    if (check_launch(h, "encode_tokens_kernel")) return 1;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ contigs -> windows
// Plan (contigs.cuh): count pass -> scan -> one D2H of the total -> capacity check -> write pass.  Scratch: the caller's
// d_win_offsets only, so a too-small capacity is reported before anything is written to d_win_start / d_win_len.
// gnm_contig_windows is the stride-6000 call of the same kernels as gnm_contig_windows_stride.
static int plan_contig_windows(gnm_handle* h, const char* fn, const uint8_t* d_seq, const int64_t* d_seq_offsets, int n_contigs,
                               int single_window, int stride, bool reverse, int64_t* d_win_start, int32_t* d_win_len,
                               int64_t capacity, int32_t* d_win_offsets, int64_t* h_n_windows, void* stream) {
  const std::string f(fn);
  if (!h) return fail(f + ": null handle");
  if (n_contigs < 0) return fail(f + ": negative contig count");
  if (capacity < 0) return fail(f + ": negative capacity");
  if (stride < 1 || stride > kWindow) return fail(f + ": stride must be in [1, 6000], not " + std::to_string(stride));
  if (!d_seq_offsets || !d_win_offsets || !h_n_windows || (n_contigs > 0 && !d_seq) ||
      (capacity > 0 && (!d_win_start || !d_win_len)))
    return fail(f + ": null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  *h_n_windows = 0;
  if (n_contigs == 0) {
    GNM_CUDA(cudaMemsetAsync(d_win_offsets, 0, sizeof(int32_t), st));
    GNM_CUDA(cudaStreamSynchronize(st));
    return 0;
  }
  const int step = single_window ? 0 : stride;         // 0: the first window only
  if (reverse) contig_plan_rc_kernel<false><<<n_contigs, kPlanThreads, 0, st>>>(d_seq, d_seq_offsets, step, d_win_offsets, nullptr, nullptr);
  else contig_plan_kernel<false><<<n_contigs, kPlanThreads, 0, st>>>(d_seq, d_seq_offsets, step, d_win_offsets, nullptr, nullptr);
  if (check_launch(h, "contig_plan_kernel<count>")) return 1;
  contig_scan_kernel<<<1, kScanThreads, 0, st>>>(d_win_offsets, n_contigs);
  if (check_launch(h, "contig_scan_kernel")) return 1;
  int32_t total = 0;
  GNM_CUDA(cudaMemcpyAsync(&total, d_win_offsets + n_contigs, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  GNM_CUDA(cudaStreamSynchronize(st));
  if (total == kPlanBadOffsets) return fail(f + ": d_seq_offsets is not non-decreasing");
  if (total == kPlanOverflow) return fail(f + ": the contigs have more than 2^31-1 windows");
  *h_n_windows = total;
  if (total > capacity)
    return fail(f + ": the contigs have " + std::to_string(total) + " windows, capacity is " + std::to_string(capacity) +
                " (n_contigs + total_bytes / " + std::to_string(stride) + " is always enough)");
  if (total == 0) return 0;
  if (reverse)
    contig_plan_rc_kernel<true><<<n_contigs, kPlanThreads, 0, st>>>(d_seq, d_seq_offsets, step, d_win_offsets, d_win_start, d_win_len);
  else
    contig_plan_kernel<true><<<n_contigs, kPlanThreads, 0, st>>>(d_seq, d_seq_offsets, step, d_win_offsets, d_win_start, d_win_len);
  return check_launch(h, "contig_plan_kernel<write>");
}

extern "C" int gnm_contig_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_seq_offsets, int n_contigs,
                                  int single_window, int64_t* d_win_start, int32_t* d_win_len, int64_t capacity,
                                  int32_t* d_win_offsets, int64_t* h_n_windows, void* stream) {
  return plan_contig_windows(h, "gnm_contig_windows", d_seq, d_seq_offsets, n_contigs, single_window, kWindow, false,
                             d_win_start, d_win_len, capacity, d_win_offsets, h_n_windows, stream);
}

extern "C" int gnm_contig_windows_stride(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_seq_offsets, int n_contigs,
                                         int stride, int64_t* d_win_start, int32_t* d_win_len, int64_t capacity,
                                         int32_t* d_win_offsets, int64_t* h_n_windows, void* stream) {
  return plan_contig_windows(h, "gnm_contig_windows_stride", d_seq, d_seq_offsets, n_contigs, 0, stride, false, d_win_start,
                             d_win_len, capacity, d_win_offsets, h_n_windows, stream);
}

extern "C" int gnm_contig_windows_rc(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_seq_offsets, int n_contigs,
                                     int single_window, int stride, int64_t* d_win_start, int32_t* d_win_len, int64_t capacity,
                                     int32_t* d_win_offsets, int64_t* h_n_windows, void* stream) {
  return plan_contig_windows(h, "gnm_contig_windows_rc", d_seq, d_seq_offsets, n_contigs, single_window, stride, true,
                             d_win_start, d_win_len, capacity, d_win_offsets, h_n_windows, stream);
}

static int launch_gather_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                                 uint8_t* d_ascii, cudaStream_t st, bool rc = false) {
  if (rc) {
    gather_windows_rc_kernel<<<n, kGatherThreads, 0, st>>>(d_seq, d_win_start, d_win_len, d_ascii);
    return check_launch(h, "gather_windows_rc_kernel");
  }
  gather_windows_kernel<<<n, kGatherThreads, 0, st>>>(d_seq, d_win_start, d_win_len, d_ascii);
  return check_launch(h, "gather_windows_kernel");
}

static int gather_windows(gnm_handle* h, const char* fn, const uint8_t* d_seq, const int64_t* d_win_start,
                          const int32_t* d_win_len, int n, uint8_t* d_ascii, void* stream, bool rc) {
  const std::string f(fn);
  if (!h) return fail(f + ": null handle");
  if (n < 0) return fail(f + ": negative window count");
  if (n == 0) return 0;
  if (!d_seq || !d_win_start || !d_win_len || !d_ascii) return fail(f + ": null buffer");
  if (reinterpret_cast<uintptr_t>(d_ascii) % 16) return fail(f + ": d_ascii must be 16-byte aligned");
  GNM_CUDA(cudaSetDevice(h->device));
  return launch_gather_windows(h, d_seq, d_win_start, d_win_len, n, d_ascii, static_cast<cudaStream_t>(stream), rc);
}
extern "C" int gnm_gather_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                                  uint8_t* d_ascii, void* stream) {
  return gather_windows(h, "gnm_gather_windows", d_seq, d_win_start, d_win_len, n, d_ascii, stream, false);
}
extern "C" int gnm_gather_windows_rc(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len,
                                     int n, uint8_t* d_ascii, void* stream) {
  return gather_windows(h, "gnm_gather_windows_rc", d_seq, d_win_start, d_win_len, n, d_ascii, stream, true);
}

// Steps of max_batch windows: gather into in_stage[step parity], then the unchanged forward step.  The gather runs on the
// step's main stream, ahead of the layer-1 kernel that reads the stage, so the TailOverlap ordering covers both buffers.
static int forward_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                           float* d_probs, float* d_embed, void* stream, bool rc = false) {
  if (!h) return fail("gnm_forward_windows: null handle");
  if (n < 0) return fail("gnm_forward_windows: negative window count");
  if (n == 0) return 0;
  if (!d_seq || !d_win_start || !d_win_len || (!d_probs && !d_embed)) return fail("gnm_forward_windows: null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  if (check_device_status(h)) return 1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TailOverlap ov(h, st, (n + h->max_batch - 1) / h->max_batch);
  for (int i = 0, off = 0; off < n; ++i, off += h->max_batch) {
    const int m = std::min(h->max_batch, n - off);
    uint8_t* stage = h->in_stage[i & 1];
    timer_mark(h, rc ? "gather_windows_rc" : "gather_windows", st);
    if (launch_gather_windows(h, d_seq, d_win_start + off, d_win_len + off, m, stage, st, rc)) return 1;
    if (ov.step(stage, nullptr, m, probs_at(d_probs, off), embed_at(d_embed, off))) return 1;
  }
  return ov.join();
}
extern "C" int gnm_forward_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len,
                                   int n, float* d_probs, void* stream) {
  return forward_windows(h, d_seq, d_win_start, d_win_len, n, d_probs, nullptr, stream);
}
extern "C" int gnm_embed_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len,
                                 int n, float* d_probs, float* d_embed, void* stream) {
  if (!d_embed && n > 0) return fail("gnm_embed_windows: d_embed is null");
  return forward_windows(h, d_seq, d_win_start, d_win_len, n, d_probs, d_embed, stream);
}
extern "C" int gnm_forward_windows_rc(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len,
                                      int n, float* d_probs, void* stream) {
  return forward_windows(h, d_seq, d_win_start, d_win_len, n, d_probs, nullptr, stream, true);
}
extern "C" int gnm_embed_windows_rc(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len,
                                    int n, float* d_probs, float* d_embed, void* stream) {
  if (!d_embed && n > 0) return fail("gnm_embed_windows_rc: d_embed is null");
  return forward_windows(h, d_seq, d_win_start, d_win_len, n, d_probs, d_embed, stream, true);
}

static int segment_any(gnm_handle* h, const float* d_probs, const int32_t* d_offsets, int n_contigs, float* d_out,
                       void* stream, bool mean) {
  if (!h) return fail("null handle");
  if (n_contigs < 0) return fail("negative contig count");
  if (n_contigs == 0) return 0;
  if (!d_probs || !d_offsets || !d_out) return fail("null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = (n_contigs + 127) / 128;
  if (mean) segment_reduce_kernel<true><<<grid, 128, 0, st>>>(d_probs, d_offsets, n_contigs, d_out);
  else segment_reduce_kernel<false><<<grid, 128, 0, st>>>(d_probs, d_offsets, n_contigs, d_out);
  return check_launch(h, "segment_reduce_kernel");
}
extern "C" int gnm_segment_mean(gnm_handle* h, const float* d_probs, const int32_t* d_offsets, int n_contigs,
                                float* d_mean, void* stream) {
  return segment_any(h, d_probs, d_offsets, n_contigs, d_mean, stream, true);
}
extern "C" int gnm_segment_sum(gnm_handle* h, const float* d_probs, const int32_t* d_offsets, int n_contigs,
                               float* d_sum4, void* stream) {
  return segment_any(h, d_probs, d_offsets, n_contigs, d_sum4, stream, false);
}

// carry_out is copied from the last segment's sum after the kernel, in stream order, so it may alias carry_in
extern "C" int gnm_segment_sum_rows(gnm_handle* h, const float* d_rows, const int32_t* d_offsets, int k, const float* d_carry_in,
                                    float* d_sums, float* d_carry_out, void* stream) {
  if (!h) return fail("gnm_segment_sum_rows: null handle");
  if (k < 0) return fail("gnm_segment_sum_rows: negative segment count");
  if (k == 0) return 0;
  if (!d_offsets || !d_sums) return fail("gnm_segment_sum_rows: null buffer");
  if ((reinterpret_cast<uintptr_t>(d_rows) | reinterpret_cast<uintptr_t>(d_sums) | reinterpret_cast<uintptr_t>(d_carry_in)) % 16)
    return fail("gnm_segment_sum_rows: d_rows, d_sums and d_carry_in must be 16-byte aligned");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  segment_sum_rows_kernel<<<k, kSegRowThreads, 0, st>>>(d_rows, d_offsets, d_carry_in, d_sums);
  if (check_launch(h, "segment_sum_rows_kernel")) return 1;
  if (d_carry_out)
    GNM_CUDA(cudaMemcpyAsync(d_carry_out, d_sums + static_cast<size_t>(k - 1) * kHidden, kHidden * sizeof(float),
                             cudaMemcpyDeviceToDevice, st));
  return 0;
}

// Wait for the work queued on `stream` and report device-side failures of the steps run so far (mbarrier time-outs,
// activation range overflow).  The asynchronous entry points only see such a flag on the NEXT call.
extern "C" int gnm_check_status(gnm_handle* h, void* stream) {
  if (!h) return fail("null handle");
  GNM_CUDA(cudaSetDevice(h->device));
  GNM_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  return check_device_status(h);
}

// Host buffers in, host buffers out; H2D of step i+1 overlaps compute of step i.  d_embed (device, or null): embeddings too.
static int classify_host(gnm_handle* h, const uint8_t* h_ascii, int n, float* h_probs, float* d_embed) {
  if (!h) return fail("null handle");
  if (n < 0) return fail("negative window count");
  if (n == 0) return 0;
  if (!h_ascii || (!h_probs && !d_embed)) return fail("null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  if (check_device_status(h)) return 1;
  const int mb = h->max_batch;
  const int steps = (n + mb - 1) / mb;
  TailOverlap ov(h, h->compute_stream, steps);
  for (int i = 0; i < steps; ++i) {
    const int b = i & 1;
    const int off = i * mb;
    const int m = std::min(mb, n - off);
    if (i >= 2) GNM_CUDA(cudaStreamWaitEvent(h->copy_stream, h->in_free[b], 0));
    GNM_CUDA(cudaMemcpyAsync(h->in_stage[b], h_ascii + static_cast<size_t>(off) * kWindow,
                             static_cast<size_t>(m) * kWindow, cudaMemcpyHostToDevice, h->copy_stream));
    GNM_CUDA(cudaEventRecord(h->in_ready[b], h->copy_stream));
    GNM_CUDA(cudaStreamWaitEvent(h->compute_stream, h->in_ready[b], 0));
    cudaStream_t tail = h->compute_stream;               // the stream that produced out_stage[b] (tail_stream when overlapped)
    if (ov.step(h->in_stage[b], nullptr, m, h_probs ? h->out_stage[b] : nullptr, embed_at(d_embed, off), &tail)) return 1;
    // the input stage is only read by layer 1, but the event sits after the step's main part (the same stream); the output
    // stage of parity b is rewritten by the tail of step i+2, which is ordered after this copy on the same stream
    GNM_CUDA(cudaEventRecord(h->in_free[b], h->compute_stream));
    if (h_probs)
      GNM_CUDA(cudaMemcpyAsync(h_probs + static_cast<size_t>(off) * 3, h->out_stage[b], static_cast<size_t>(m) * 3 * sizeof(float),
                               cudaMemcpyDeviceToHost, tail));
    if (ov.on) GNM_CUDA(cudaEventRecord(h->tail_done[b], tail));     // re-record: the buffer set is free once the copy is queued behind the tail
  }
  if (ov.join()) return 1;
  GNM_CUDA(cudaStreamSynchronize(h->compute_stream));
  if (ov.on) GNM_CUDA(cudaStreamSynchronize(h->tail_stream));
  return check_device_status(h);
}
extern "C" int gnm_classify_host(gnm_handle* h, const uint8_t* h_ascii, int n, float* h_probs) {
  return classify_host(h, h_ascii, n, h_probs, nullptr);
}
extern "C" int gnm_embed_host(gnm_handle* h, const uint8_t* h_ascii, int n, float* h_probs, float* d_embed) {
  if (!d_embed && n > 0) return fail("gnm_embed_host: d_embed is null");
  return classify_host(h, h_ascii, n, h_probs, d_embed);
}

// ------------------------------------------------------------------------------------------------
extern "C" int gnm_set_option(gnm_handle* h, const char* name, int value) {
  if (!h || !name) return fail("null argument");
  const std::string k(name);
  if (k == "conv_impl") { if (value != 0 && value != 1) return fail("conv_impl must be 0 or 1"); h->conv_impl = value; }
  else if (k == "debug_stop") h->debug_stop = value;
  else if (k == "conv_experiment") h->conv_experiment = value;
  else if (k == "fuse_l1") h->fuse_l1 = value ? 1 : 0;
  else if (k == "fuse_gather") h->fuse_gather = value ? 1 : 0;
  else if (k == "tail_overlap") h->tail_overlap = value ? 1 : 0;
  else if (k == "wv_cost_group") {      // experiment: per-mille cost of one position group per warp in wv_split's unit cost model (base = 1000)
    if (value < 0 || value > 10000) return fail("wv_cost_group must be in [0, 10000]");
    h->wv_cost_group = value * 1e-3f; h->split_groups[0] = h->split_groups[1] = -1;
  }
  else if (k == "conv_cluster") { if (value != 1 && value != 2 && value != 4 && value != 8) return fail("conv_cluster must be 1, 2, 4 or 8"); h->conv_cluster = value; }
  else if (k == "profile_stages") { h->profile_stages = value ? 1 : 0; h->timer.names.clear(); }   // (re)starts the record
  else return fail("unknown option: " + k);
  return 0;
}
extern "C" int gnm_get_option(gnm_handle* h, const char* name, int* value) {
  if (!h || !name || !value) return fail("null argument");
  const std::string k(name);
  if (k == "conv_impl") *value = h->conv_impl;
  else if (k == "debug_stop") *value = h->debug_stop;
  else if (k == "profile_stages") *value = h->profile_stages;
  else if (k == "fuse_l1") *value = h->fuse_l1;
  else if (k == "fuse_gather") *value = h->fuse_gather;
  else if (k == "tail_overlap") *value = h->tail_overlap;
  else if (k == "max_batch") *value = h->max_batch;
  else if (k == "num_sms") *value = h->num_sms;
  else return fail("unknown option: " + k);
  return 0;
}
extern "C" long long gnm_kernel_launches(gnm_handle* h) { return h ? h->launches : 0; }

extern "C" int gnm_stage_times(gnm_handle* h, const char** names, float* ms, int* count) {
  if (!h || !count) return fail("null argument");
  GNM_CUDA(cudaSetDevice(h->device));
  const int ns = static_cast<int>(h->timer.names.size());
  const int cap = *count;
  *count = 0;
  if (ns < 2) return 0;
  GNM_CUDA(cudaEventSynchronize(h->timer.events[ns - 1]));
  int k = 0;
  for (int i = 0; i + 1 < ns && k < cap; ++i) {
    if (std::strcmp(h->timer.names[i], "end") == 0) continue;     // gap between two recorded steps
    float t = 0.f;
    GNM_CUDA(cudaEventElapsedTime(&t, h->timer.events[i], h->timer.events[i + 1]));
    if (names) names[k] = h->timer.names[i];
    if (ms) ms[k] = t;
    ++k;
  }
  *count = k;
  return 0;
}

static int attr_debug_fetch(gnm_handle* h, const gnm_attr* a, const std::string& k, int n, float* d_dst, cudaStream_t st);

extern "C" int gnm_debug_fetch(gnm_handle* h, const char* which, int n, float* d_dst, void* stream) {
  if (!h || !which || !d_dst) return fail("null argument");
  if (n < 1 || n > h->max_batch) return fail("gnm_debug_fetch: n out of range");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const std::string k(which);
  const float* src = nullptr;
  size_t count = 0;
  if ((k.rfind("route", 0) == 0 || k.rfind("attr_", 0) == 0) && n > h->attr_mb)   // the last attribution context's buffers
    return fail("gnm_debug_fetch: n exceeds the max_batch of the last attribution call's context (" + std::to_string(h->attr_mb) + ")");
  if (k == "buf0" || k == "buf1") {
    const size_t rows = static_cast<size_t>(n) * kTok;
    join_rows_kernel<<<static_cast<unsigned>((rows * kC + 255) / 256), 256, 0, st>>>(h->ybuf[k == "buf1"], d_dst, rows,
                                                                                     h->ybuf_fp8lo[k == "buf1"]);
    return check_launch(h, "join_rows_kernel");
  } else if (k == "q0" || k == "q1") { src = h->q[k == "q1"]; count = static_cast<size_t>(n) * kPooled * kC; }
  else if (k == "mpi0" || k == "mpi1") { src = h->mpi[k == "mpi1"]; count = static_cast<size_t>(n) * kPatches; }
  else if (k == "h0") { src = h->h0; count = static_cast<size_t>(n) * 256; }
  else if (k == "h1" || k == "h2") { src = k == "h1" ? h->h1 : h->h2; count = static_cast<size_t>(n) * kHidden; }
  else if (k == "logits") { src = h->logits; count = static_cast<size_t>(n) * kLogitsLd; }
  else if (k == "conv_dbg") { src = reinterpret_cast<const float*>(h->conv_dbg); count = static_cast<size_t>(h->num_sms) * 16; }
  else if (k == "route0" || k == "route1") {               // uint8 [n][749][128]: n * 749 * 128 BYTES
    const uint8_t* r = h->attr_route[k == "route1"];
    if (!r) return fail("gnm_debug_fetch: no attribution call has run on this handle");
    GNM_CUDA(cudaMemcpyAsync(d_dst, r, static_cast<size_t>(n) * kPooled * kC, cudaMemcpyDeviceToDevice, st));
    return 0;
  } else if (k == "routeq0" || k == "routeq1") {
    src = h->attr_rq[k == "routeq1"];
    if (!src) return fail("gnm_debug_fetch: no attribution call has run on this handle");
    count = static_cast<size_t>(n) * kPooled * kC;
  } else if (k.rfind("attr_", 0) == 0) {
    if (!h->attr_last) return fail("gnm_debug_fetch: no attribution call has run on this handle");
    return attr_debug_fetch(h, h->attr_last, k, n, d_dst, st);
  }
  else return fail("gnm_debug_fetch: unknown buffer " + k);
  GNM_CUDA(cudaMemcpyAsync(d_dst, src, count * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// A classifier head (gnm_head_create): its dense_1 with BN folded into scale / shift, dense_1 as TF32 halves for the tensor
// cores, dense_2.
struct gnm_head {
  int C = 0;
  std::vector<void*> allocs;
  float *d1w = nullptr, *d1b = nullptr, *scale = nullptr, *shift = nullptr, *dwT_hi = nullptr, *dwT_lo = nullptr;
  float *d2w = nullptr, *d2b = nullptr;
  CUtensorMap tm_b[2];
  double *nv_center = nullptr, *nv_whitening = nullptr, *nv_means = nullptr;   // novelty model (gnm_head_set_novelty)
};

// The head on the tensor cores from the TF32 halves of its input in hA_hi[1] / hA_lo[1] (dense layer 0's epilogue leaves h1's
// there; gnm_head_forward splits the embeddings into them): dense_1 + BN + ReLU -> h2, then the C-class softmax -> d_probs.
static int head_forward_tc(gnm_handle* h, const gnm_head* hd, int n, float* d_probs, cudaStream_t st) {
  if (launch_dense_tc_maps(h, h->tm_hd_a[1], hd->tm_b, kHidden, n, hd->d1b, hd->scale, hd->shift, h->h2, nullptr, nullptr, nullptr,
                           st)) return 1;
  head_softmax_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(h->h2, hd->d2w, hd->d2b, d_probs, n, hd->C);
  return check_launch(h, "head_softmax_kernel");
}

// ------------------------------------------------------------------------------------------------ attributions (attr.cuh)
// Workspace of the attribution pass, separate from the handle so that plain handles keep their memory.  Per window:
// y1 copy, g_z3 and g_z2 operand rows (3 x 4.6 MB), fp32 g_y1 / g_z rows (2 x 3.1 MB), routing + routed maxima (2 x 0.48 MB):
// ~21 MB (gnm_attr_bytes_per_window).
struct gnm_attr {
  gnm_handle* h = nullptr;
  int max_batch = 0;
  uint8_t* y1 = nullptr;                                // layer 1 re-run: the forward's y1 (ybuf[0] is overwritten by conv3)
  uint8_t* gz3 = nullptr; uint8_t* gz2 = nullptr;       // conv operand rows of s_w g_z3, s_w g_z2, time-reversed
  float* f32a = nullptr;                                // fp32 rows: g_z3, then s_w g_z2 (each before packing), then s_w g_z1
  float* gy1 = nullptr;                                 // fp32 rows: IGLOO#0's part of g_y1
  uint8_t* route[2] = {nullptr, nullptr}; float* rq[2] = {nullptr, nullptr};
  float* g_out = nullptr; float* alpha = nullptr; float* g_logit = nullptr; float* g_mpi = nullptr;
  float* blockmax = nullptr; float* s_w = nullptr; float* probs = nullptr;
  float* unitmax = nullptr; float* s2 = nullptr;        // conv3 backward: max |s_w g_z2| per unit and warp; its power of two
  double* nv_r = nullptr; float* nv_g = nullptr;        // novelty attributions: fp64 r = P (h1 - center) - m_c, fp32 g_h1
  int32_t* nv_target = nullptr;                         //   each row's target class (uploaded per chunk)
  float* nv_base = nullptr;                             //   the IG baseline's distances [C]
  uint8_t* wpackT[2] = {nullptr, nullptr};              // W2^T, W3^T packed like the forward's conv weights
  float out_scaleT[2] = {1.f, 1.f};
  float* wvT[2] = {nullptr, nullptr}; float* wqkT[2] = {nullptr, nullptr};
  int32_t* pos_start[2] = {nullptr, nullptr}; int32_t* slot_patch[2] = {nullptr, nullptr};
  CUtensorMap tm_y1, tm_gz3, tm_gz2, tm_wT[2];
  std::vector<void*> allocs;
};

static int attr_alloc(gnm_attr* a, void** p, size_t bytes) {
  GNM_CUDA(cudaMalloc(p, bytes));
  a->allocs.push_back(*p);
  return 0;
}
template <class T>
static int attr_upload(gnm_attr* a, T** dst, const std::vector<T>& src) {
  if (attr_alloc(a, reinterpret_cast<void**>(dst), src.size() * sizeof(T))) return 1;
  GNM_CUDA(cudaMemcpy(*dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}
template <class T>
static int fetch_host(std::vector<T>& dst, const T* src, size_t count) {
  dst.resize(count);
  GNM_CUDA(cudaMemcpy(dst.data(), src, count * sizeof(T), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int gnm_attr_destroy(gnm_attr* a) {
  if (!a) return 0;
  cudaSetDevice(a->h->device);
  cudaDeviceSynchronize();
  for (int s = 0; s < 2; ++s)
    if (a->h->attr_route[s] == a->route[s]) {
      a->h->attr_route[s] = nullptr; a->h->attr_rq[s] = nullptr; a->h->attr_last = nullptr;
      a->h->attr_mb = 0;
    }
  for (void* p : a->allocs) cudaFree(p);
  delete a;
  return 0;
}

extern "C" int gnm_attr_create(gnm_handle* h, int max_batch, gnm_attr** out) {
  if (!h || !out) return fail("gnm_attr_create: null argument");
  *out = nullptr;
  if (max_batch < 1 || max_batch > h->max_batch)
    return fail("gnm_attr_create: max_batch must be in [1, the handle's max_batch = " + std::to_string(h->max_batch) + "]");
  GNM_CUDA(cudaSetDevice(h->device));
  gnm_attr* a = new gnm_attr();
  a->h = h;
  a->max_batch = max_batch;
  *out = a;                                             // so the caller can gnm_attr_destroy() after a partial failure
  const size_t mb = static_cast<size_t>(max_batch), rows = mb * kTok;
  void** v = nullptr;
#define ATTR_ALLOC(ptr, bytes) do { v = reinterpret_cast<void**>(&(ptr)); if (attr_alloc(a, v, (bytes))) return 1; } while (0)
  ATTR_ALLOC(a->y1, rows * kRowBytes);
  ATTR_ALLOC(a->gz3, rows * kRowBytes);
  ATTR_ALLOC(a->gz2, rows * kRowBytes);
  ATTR_ALLOC(a->f32a, rows * kC * sizeof(float));
  ATTR_ALLOC(a->gy1, rows * kC * sizeof(float));
  for (int s = 0; s < 2; ++s) {
    ATTR_ALLOC(a->route[s], mb * kPooled * kC);
    ATTR_ALLOC(a->rq[s], mb * kPooled * kC * sizeof(float));
  }
  ATTR_ALLOC(a->g_out, mb * 256 * sizeof(float));
  ATTR_ALLOC(a->alpha, mb * kLogitsLd * sizeof(float));
  ATTR_ALLOC(a->g_logit, mb * kLogitsLd * sizeof(float));
  ATTR_ALLOC(a->g_mpi, mb * kPatches * sizeof(float));
  ATTR_ALLOC(a->blockmax, mb * kAttrPosBlocks * sizeof(float));
  ATTR_ALLOC(a->s_w, mb * sizeof(float));
  ATTR_ALLOC(a->unitmax, mb * kUnitsPerWin * 8 * sizeof(float));
  ATTR_ALLOC(a->s2, mb * sizeof(float));
  ATTR_ALLOC(a->probs, mb * 3 * sizeof(float));
  ATTR_ALLOC(a->nv_r, mb * kHidden * sizeof(double));
  ATTR_ALLOC(a->nv_g, mb * kHidden * sizeof(float));
  ATTR_ALLOC(a->nv_target, mb * sizeof(int32_t));
  ATTR_ALLOC(a->nv_base, kNvMaxClasses * sizeof(float));
#undef ATTR_ALLOC
  // ---- weights, derived from the handle's device copies
  for (int L = 0; L < 2; ++L) {                         // conv2, conv3: W[j]^T in the forward's pack, same split and scale
    std::vector<float> Wk, WT(static_cast<size_t>(kTaps) * kC * kC);
    if (fetch_host(Wk, h->conv_w32[L], WT.size())) return 1;
    for (int j = 0; j < kTaps; ++j)
      for (int i = 0; i < kC; ++i)
        for (int o = 0; o < kC; ++o)
          WT[(static_cast<size_t>(j) * kC + o) * kC + i] = Wk[(static_cast<size_t>(j) * kC + i) * kC + o];
    std::vector<uint8_t> pk;
    if (pack_conv_weights(WT.data(), pk, &a->out_scaleT[L], "gnm_attr_create")) return 1;
    if (attr_upload(a, &a->wpackT[L], pk)) return 1;
  }
  for (int s = 0; s < 2; ++s) {
    std::vector<float> wv, wvT(static_cast<size_t>(kC) * kC), qk, qkT(static_cast<size_t>(kPooled) * kPatches);
    if (fetch_host(wv, h->wv32[s], wvT.size())) return 1;
    for (int k = 0; k < kC; ++k)
      for (int c = 0; c < kC; ++c) wvT[static_cast<size_t>(c) * kC + k] = wv[static_cast<size_t>(k) * kC + c];
    if (attr_upload(a, &a->wvT[s], wvT)) return 1;
    if (fetch_host(qk, h->wqk[s], qkT.size())) return 1;
    for (int i = 0; i < kPatches; ++i)
      for (int p = 0; p < kPooled; ++p) qkT[static_cast<size_t>(p) * kPatches + i] = qk[static_cast<size_t>(i) * kPooled + p];
    if (attr_upload(a, &a->wqkT[s], qkT)) return 1;
    // inverse of the gather's packing: the first 8,400 slots are the patch entries sorted by position (pack_patches)
    std::vector<int32_t> ent_pos, slot_of, pos_start(kTok + 1, 0), slot_patch(static_cast<size_t>(kPatches) * kPatchLen);
    if (fetch_host(ent_pos, h->ent_pos[s], static_cast<size_t>(kPatches) * kPatchLen)) return 1;
    if (fetch_host(slot_of, h->slot_of[s], slot_patch.size())) return 1;
    for (size_t e = 0; e < slot_of.size(); ++e) slot_patch[slot_of[e]] = static_cast<int32_t>(e / kPatchLen);
    for (int32_t p : ent_pos) pos_start[p + 1]++;
    for (int t = 0; t < kTok; ++t) pos_start[t + 1] += pos_start[t];
    if (attr_upload(a, &a->pos_start[s], pos_start)) return 1;
    if (attr_upload(a, &a->slot_patch[s], slot_patch)) return 1;
  }
  PFN_encodeTiled enc = nullptr;
  if (get_encode_fn(&enc)) return 1;
  if (make_act_map(enc, &a->tm_y1, a->y1, max_batch)) return 1;
  if (make_act_map(enc, &a->tm_gz3, a->gz3, max_batch)) return 1;
  if (make_act_map(enc, &a->tm_gz2, a->gz2, max_batch)) return 1;
  for (int L = 0; L < 2; ++L)
    if (make_w_map(enc, &a->tm_wT[L], a->wpackT[L], kConvStages, 64)) return 1;
  GNM_CUDA(cudaFuncSetAttribute(conv_t_attr_kernel<kConvRoute>, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvTSmem));
  GNM_CUDA(cudaFuncSetAttribute(conv_t_attr_kernel<kConvBwd>, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvTSmem));
  GNM_CUDA(cudaDeviceSynchronize());
  return 0;
}

// the w_v pass of IGLOO kernel s over `tm` with the routing epilogue: route[s], rq[s] (= the forward's q[s], bit for bit)
static int launch_route(gnm_handle* h, gnm_attr* a, int s, const CUtensorMap& tm, int n, cudaStream_t st) {
  ConvTcParams p;
  p.status = h->status; p.experiment = 0; p.dbg = nullptr;
  p.bias = nullptr; p.y_out = nullptr; p.q_out = a->rq[s];
  p.out_scale = h->wv_out_scale[s]; p.out_fp8 = 0;
  p.n_tiles = n * kUnitsPerWin;
  ConvAttrExt x = {};
  x.route_out = a->route[s];
  conv_t_attr_kernel<kConvRoute><<<std::min(h->num_sms, p.n_tiles), kConvThreads, kConvTSmem, st>>>(tm, h->tm_w_half[2 + s], p, x);
  return check_launch(h, "conv_t_attr_kernel<route>");
}
// backward of conv layer L (0 = conv2, 1 = conv3) over time-reversed gradient rows into fp32 rows
static int launch_conv_bwd(gnm_handle* h, gnm_attr* a, int L, const CUtensorMap& tm_in, const uint8_t* mask_rows,
                           const float* add_rows, const float* s_in, float* f32_out, float* unit_max, int n, cudaStream_t st) {
  ConvTcParams p;
  p.status = h->status; p.experiment = 0; p.dbg = nullptr;
  p.bias = nullptr; p.y_out = nullptr; p.q_out = nullptr;
  p.out_scale = a->out_scaleT[L]; p.out_fp8 = 1;
  p.n_tiles = n * kUnitsPerWin;
  ConvAttrExt x = {};
  x.mask_rows = mask_rows; x.add_rows = add_rows; x.s_w = a->s_w; x.s_in = s_in; x.f32_out = f32_out; x.unit_max = unit_max;
  conv_t_attr_kernel<kConvBwd><<<std::min(h->num_sms, p.n_tiles), kConvThreads, kConvTSmem, st>>>(tm_in, a->tm_wT[L], p, x);
  return check_launch(h, "conv_t_attr_kernel<bwd>");
}
// attention part and g_y of IGLOO kernel s (logits of s must be in h->logits)
static int launch_igloo_bwd(gnm_handle* h, gnm_attr* a, int s, int n, cudaStream_t st) {
  attr_igloo_prep_kernel<<<n, 256, 0, st>>>(h->logits, h->q[s], a->g_out + s * kC, a->alpha, a->g_logit);
  if (check_launch(h, "attr_igloo_prep_kernel")) return 1;
  if (launch_sgemm(h, a->g_logit, kLogitsLd, a->wqkT[s], kPatches, a->g_mpi, kPatches, n, kPatches, kPooled, nullptr, nullptr,
                   nullptr, 0, st)) return 1;
  IglooBwdParams P;
  P.alpha = a->alpha; P.g_out = a->g_out + s * kC; P.route = a->route[s]; P.wvT = a->wvT[s]; P.g_mpi = a->g_mpi;
  P.pos_start = a->pos_start[s]; P.slot_patch = a->slot_patch[s]; P.ent_w = h->ent_w[s];
  P.y_rows = h->ybuf[0]; P.out = s ? a->f32a : a->gy1; P.blockmax = a->blockmax;
  dim3 grid(kAttrPosBlocks, n);
  if (s) attr_igloo_backward_kernel<true><<<grid, 256, 0, st>>>(P);
  else attr_igloo_backward_kernel<false><<<grid, 256, 0, st>>>(P);
  return check_launch(h, "attr_igloo_backward_kernel");
}

// One chunk: the unchanged forward step, strictly in order, then the backward pass over the state that step left behind
// (ybuf[0] = y3, ybuf[1] = y2, q / logits of IGLOO#1, h1, h2).  With `ig`, the n rows are interpolated inputs (forward_main)
// and the layer-1 result of row r, g[t, tok[t]] (minus g[t, 0] for the N baseline), goes to the g_y1 rows as [n][5997]
// (layer1_ig_kernel); d_attr is not used.
// With a head `hd`, the gradient is that of the head's log p_c: after the forward step, the head runs on the h1 halves that
// dense layer 0's epilogue left in hA_hi[1] / hA_lo[1] (head_forward_tc, as gnm_head_forward after its split).  Its hidden rows
// replace the shipped ones in h2 and its probabilities [n][C] go to d_head_probs, or else to blockmax (376 B per window >= 128):
// both are read by attr_head_backward_kernel, and blockmax is rewritten only after it, by IGLOO#1's backward.
// With `novelty`, the gradient is instead that of the head's novelty distance D_c to each row's target class (a->nv_target,
// uploaded by the caller): r and g_h1 in fp64 on the h1 rows the forward left (nv_residual_kernel, nv_grad_kernel), then g_out
// (attr_novelty_backward_kernel); no head forward.  d_dist [n][C], when given, gets the rows' distances (nv_score_kernel).
static int attribute_step(gnm_handle* h, gnm_attr* a, const uint8_t* d_ascii, int n, int target, float* d_probs, float* d_attr,
                          cudaStream_t st, const L1Interp* ig = nullptr, const gnm_head* hd = nullptr,
                          float* d_head_probs = nullptr, bool novelty = false, float* d_dist = nullptr) {
  float* probs = d_probs ? d_probs : a->probs;
  if (forward_step(h, d_ascii, nullptr, n, probs, nullptr, st, ig)) return 1;
  float* head_probs = d_head_probs ? d_head_probs : a->blockmax;
  if (hd && !novelty) {
    timer_mark(h, "attr_head_fwd", st);
    if (head_forward_tc(h, hd, n, head_probs, st)) return 1;
  }
  dim3 egrid((kTok + kEmbSeg - 1) / kEmbSeg, n), sgrid((kTok + kAttrSeg - 1) / kAttrSeg, n);
  timer_mark(h, "attr_layer1", st);
  if (ig) {
    embed_conv1_ig_kernel<<<egrid, kEmbThreads, 0, st>>>(d_ascii, h->conv1_table, h->conv1_triple, h->conv1_bias, a->y1, ig->m,
                                                         ig->baseline, h->status);
    if (check_launch(h, "embed_conv1_ig_kernel")) return 1;
  } else {
  embed_conv1_kernel<true><<<egrid, kEmbThreads, 0, st>>>(d_ascii, nullptr, h->conv1_table, h->conv1_triple, h->conv1_bias, a->y1, n, h->status);
  if (check_launch(h, "embed_conv1_kernel")) return 1;
  }
  timer_mark(h, "attr_route1", st);
  if (launch_route(h, a, 1, h->tm_act[0], n, st)) return 1;                  // y3
  timer_mark(h, "attr_route0", st);
  if (launch_route(h, a, 0, a->tm_y1, n, st)) return 1;                      // y1
  timer_mark(h, "attr_head", st);
  if (novelty) {
    const unsigned blocks = static_cast<unsigned>((n + kNvTile - 1) / kNvTile);
    if (d_dist) {
      nv_score_kernel<<<blocks, kNvThreads, kNvScoreSmem, st>>>(h->h1, n, hd->nv_center, hd->nv_whitening, hd->nv_means, hd->C,
                                                                d_dist);
      if (check_launch(h, "nv_score_kernel")) return 1;
    }
    nv_residual_kernel<<<blocks, kNvThreads, 0, st>>>(h->h1, n, hd->nv_center, hd->nv_whitening, hd->nv_means, a->nv_target,
                                                      a->nv_r);
    if (check_launch(h, "nv_residual_kernel")) return 1;
    nv_grad_kernel<<<dim3(blocks, kNvTiles), kNvThreads, 0, st>>>(a->nv_r, n, hd->nv_whitening, a->nv_g);
    if (check_launch(h, "nv_grad_kernel")) return 1;
    attr_novelty_backward_kernel<<<n, 256, 0, st>>>(a->nv_g, h->h1, h->d0w, h->bn0_scale, a->g_out);
    if (check_launch(h, "attr_novelty_backward_kernel")) return 1;
  } else {
    if (hd)
      attr_head_backward_kernel<<<n, 256, 0, st>>>(head_probs, h->h1, h->h2, hd->d2w, hd->d1w, hd->scale, h->d0w,
                                                   h->bn0_scale, attr_classes(target, hd->C), a->g_out);
    else
      attr_head_backward_kernel<<<n, 256, 0, st>>>(probs, h->h1, h->h2, h->d2w, h->d1w, h->bn1_scale, h->d0w, h->bn0_scale,
                                                   attr_classes(target, 3), a->g_out);
    if (check_launch(h, "attr_head_backward_kernel")) return 1;
  }
  timer_mark(h, "attr_igloo1", st);
  if (launch_igloo_bwd(h, a, 1, n, st)) return 1;                            // -> fp32 g_z3, block maxima
  attr_pack_kernel<<<sgrid, 256, 0, st>>>(a->f32a, a->blockmax, a->s_w, a->gz3);
  if (check_launch(h, "attr_pack_kernel")) return 1;
  timer_mark(h, "attr_conv3_bwd", st);
  if (launch_conv_bwd(h, a, 1, a->tm_gz3, h->ybuf[1], nullptr, nullptr, a->f32a, a->unitmax, n, st)) return 1;   // mask y2 -> s_w g_z2
  attr_pack_gz2_kernel<<<sgrid, 256, 0, st>>>(a->f32a, a->unitmax, a->s2, a->gz2, h->status);      // s2 s_w g_z2
  if (check_launch(h, "attr_pack_gz2_kernel")) return 1;
  timer_mark(h, "attr_igloo0", st);
  if (launch_logits(h, 0, n, st)) return 1;                                  // IGLOO#0's logits (the tail overwrote them)
  if (launch_igloo_bwd(h, a, 0, n, st)) return 1;                            // -> fp32 g_y1 (IGLOO#0 part)
  timer_mark(h, "attr_conv2_bwd", st);
  if (launch_conv_bwd(h, a, 0, a->tm_gz2, a->y1, a->gy1, a->s2, a->f32a, nullptr, n, st)) return 1;   // / s2, + s_w g_y1, mask y1 -> s_w g_z1
  timer_mark(h, "attr_layer1_attr", st);
  if (ig) {
    layer1_ig_kernel<<<sgrid, 256, 0, st>>>(d_ascii, a->f32a, h->conv1_table, a->s_w, ig->m, ig->baseline, a->gy1);
    if (check_launch(h, "layer1_ig_kernel")) return 1;
  } else {
  layer1_attr_kernel<<<sgrid, 256, 0, st>>>(d_ascii, a->f32a, h->conv1_table, a->s_w, d_attr);
  if (check_launch(h, "layer1_attr_kernel")) return 1;
  }
  timer_mark(h, "end", st);
  for (int s = 0; s < 2; ++s) { h->attr_route[s] = a->route[s]; h->attr_rq[s] = a->rq[s]; }
  h->attr_last = a;
  h->attr_mb = a->max_batch;
  return 0;
}

// gnm_debug_fetch's "attr_*" buffers of the last attribution chunk (include/gnm.h); n <= the context's max_batch (checked)
static int attr_debug_fetch(gnm_handle* h, const gnm_attr* a, const std::string& k, int n, float* d_dst, cudaStream_t st) {
  const size_t rows = static_cast<size_t>(n) * kTok;
  const float* src = nullptr;
  size_t count = 0;
  if (k == "attr_gz3" || k == "attr_gz2") {                // operand rows, time-reversed: joined, back in position order
    const uint8_t* r = k == "attr_gz3" ? a->gz3 : a->gz2;
    join_rows_kernel<<<static_cast<unsigned>((rows * kC + 255) / 256), 256, 0, st>>>(r, d_dst, rows, 1);
    if (check_launch(h, "join_rows_kernel")) return 1;
    reverse_rows_kernel<<<static_cast<unsigned>((rows * kC / 2 + 255) / 256), 256, 0, st>>>(d_dst, n);
    return check_launch(h, "reverse_rows_kernel");
  }
  if (k == "attr_g_out") { src = a->g_out; count = static_cast<size_t>(n) * 256; }
  else if (k == "attr_g_h1") { src = a->nv_g; count = static_cast<size_t>(n) * kHidden; }
  else if (k == "attr_s_w") { src = a->s_w; count = n; }
  else if (k == "attr_s2") { src = a->s2; count = n; }
  else if (k == "attr_gy1") { src = a->gy1; count = rows * kC; }
  else if (k == "attr_gz1") { src = a->f32a; count = rows * kC; }
  else if (k == "attr_y1") {
    join_rows_kernel<<<static_cast<unsigned>((rows * kC + 255) / 256), 256, 0, st>>>(a->y1, d_dst, rows, 0);
    return check_launch(h, "join_rows_kernel");
  }
  else return fail("gnm_debug_fetch: unknown buffer " + k);
  GNM_CUDA(cudaMemcpyAsync(d_dst, src, count * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// the target check of the attribution calls: the shipped classes, or [0, C) of a head
static int check_target(const std::string& f, const gnm_head* hd, int target) {
  if (!hd) {
    if (target < 0 || target > 2) return fail(f + ": target must be 0 (chromosome), 1 (plasmid) or 2 (virus)");
  } else if (target < 0 || target >= hd->C) {
    return fail(f + ": target must be a class of the head, in [0, " + std::to_string(hd->C) + "), not " + std::to_string(target));
  }
  return 0;
}

// The novelty attribution calls' own arguments: HOST targets [n], DEVICE distances [n][C] and (IG) [n][2], each or NULL.
struct NvAttrArgs {
  const int32_t* h_target;
  float* d_dist;
  float* d_dist_target;
};

// the checks of the novelty attribution calls, before any launch: the head carries a model and every target is a class of it
static int check_novelty(const std::string& f, const gnm_head* hd, const NvAttrArgs* nv, int n) {
  if (!hd->nv_center) return fail(f + ": the head has no novelty model (gnm_head_set_novelty)");
  if (n > 0 && !nv->h_target) return fail(f + ": null target array");
  for (int i = 0; i < n; ++i)
    if (nv->h_target[i] < 0 || nv->h_target[i] >= hd->C)
      return fail(f + ": target[" + std::to_string(i) + "] = " + std::to_string(nv->h_target[i]) +
                  " is not a class of the head, in [0, " + std::to_string(hd->C) + ")");
  GNM_CUDA(cudaFuncSetAttribute(nv_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kNvScoreSmem));
  return 0;
}

// targets of windows [0, m) of h_target, each repeated for its `rows` rows, to the context's target list (stream-ordered behind
// the previous chunk's readers).  A copy from pageable memory may make the host wait for the stream first: 4 B per row, one
// copy per chunk of up to 256 rows, so each chunk's launches are issued once the previous chunk has run.
static int upload_targets(gnm_attr* a, const int32_t* h_target, int m, int rows, cudaStream_t st) {
  std::vector<int32_t> v(static_cast<size_t>(m) * rows);
  for (size_t i = 0; i < v.size(); ++i) v[i] = h_target[i / rows];
  GNM_CUDA(cudaMemcpyAsync(a->nv_target, v.data(), v.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  return 0;
}

static int attribute_any(gnm_handle* h, gnm_attr* a, const char* fn, const uint8_t* d_ascii, const uint8_t* d_seq,
                         const int64_t* d_win_start, const int32_t* d_win_len, int n, int target, float* d_probs, float* d_attr,
                         void* stream, const gnm_head* hd = nullptr, float* d_head_probs = nullptr,
                         const NvAttrArgs* nv = nullptr) {
  const std::string f(fn);
  if (!h || !a) return fail(f + ": null handle or attribution context");
  if (a->h != h) return fail(f + ": the attribution context belongs to another handle");
  if (n < 0) return fail(f + ": negative window count");
  if (nv ? check_novelty(f, hd, nv, n) : check_target(f, hd, target)) return 1;
  if (h->conv_impl != 0)
    return fail(f + ": attributions need the tensor-core path (conv_impl = 0); the fp32 validation kernels have no backward pass");
  if (h->debug_stop != 0) return fail(f + ": debug_stop must be 0");
  if (n == 0) return 0;
  if (!d_attr || (!d_ascii && (!d_seq || !d_win_start || !d_win_len))) return fail(f + ": null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  if (check_device_status(h)) return 1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int off = 0; off < n; off += a->max_batch) {
    const int m = std::min(a->max_batch, n - off);
    const uint8_t* asc = d_ascii ? d_ascii + static_cast<size_t>(off) * kWindow : h->in_stage[0];
    if (!d_ascii && launch_gather_windows(h, d_seq, d_win_start + off, d_win_len + off, m, h->in_stage[0], st)) return 1;
    float* head_probs = d_head_probs ? d_head_probs + static_cast<size_t>(off) * hd->C : nullptr;
    float* dist = nv && nv->d_dist ? nv->d_dist + static_cast<size_t>(off) * hd->C : nullptr;
    if (nv && upload_targets(a, nv->h_target + off, m, 1, st)) return 1;
    if (attribute_step(h, a, asc, m, target, probs_at(d_probs, off), d_attr + static_cast<size_t>(off) * kTok, st, nullptr, hd,
                       head_probs, nv != nullptr, dist)) return 1;
  }
  return 0;
}

extern "C" int gnm_attribute_ascii(gnm_handle* h, gnm_attr* a, const uint8_t* d_ascii, int n, int target, float* d_probs,
                                   float* d_attr, void* stream) {
  if (n > 0 && !d_ascii) return fail("gnm_attribute_ascii: null buffer");
  return attribute_any(h, a, "gnm_attribute_ascii", d_ascii, nullptr, nullptr, nullptr, n, target, d_probs, d_attr, stream);
}
extern "C" int gnm_attribute_windows(gnm_handle* h, gnm_attr* a, const uint8_t* d_seq, const int64_t* d_win_start,
                                     const int32_t* d_win_len, int n, int target, float* d_probs, float* d_attr, void* stream) {
  if (n > 0 && (!d_seq || !d_win_start || !d_win_len)) return fail("gnm_attribute_windows: null buffer");
  return attribute_any(h, a, "gnm_attribute_windows", nullptr, d_seq, d_win_start, d_win_len, n, target, d_probs, d_attr, stream);
}
// ------------------------------------------------------------------------------------------------ integrated gradients
// Chunks of floor(max_batch / steps) windows, so that a window's `steps` rows never span chunks.  Per chunk, in order:
//   1. the unchanged forward of the windows: probabilities (bitwise gnm_forward_*) and log p_c(x);
//   2. attribute_step over the windows x steps rows (row w steps + k: window w at alpha_k), layer-1 results to the g_y1 rows;
//   3. ig_reduce_kernel: IG = the rows' mean over k, ascending.
// log p_c(x') is the same for every window: one one-row forward of the baseline per call, before the first chunk (only when
// d_logp is given), so the debug buffers still hold the last chunk's rows afterwards.
// attribute_ig_any's chunk loop for a head's novelty distance (checked by the caller): the same chunks, rows and mean over k,
// with D_c in place of log p_c.  D_c(x') comes from the baseline's one-row forward before the first chunk, D_c(x) from each
// chunk's own forward (bitwise gnm_head_novelty of the window's embedding); each window's target is repeated over its rows.
static int attribute_novelty_ig(gnm_handle* h, gnm_attr* a, const uint8_t* d_ascii, const uint8_t* d_seq,
                                const int64_t* d_win_start, const int32_t* d_win_len, int n, int steps, int baseline,
                                float* d_probs, float* d_attr, cudaStream_t st, const gnm_head* hd, const NvAttrArgs* nv) {
  const int per = a->max_batch / steps, C = hd->C;
  if (nv->d_dist_target) {                                      // the baseline's distances to every class, a->nv_base [C]
    const L1Interp base = {0, baseline};
    if (forward_step(h, d_ascii ? d_ascii : h->in_stage[0], nullptr, 1, a->probs, nullptr, st, &base)) return 1;
    nv_score_kernel<<<1, kNvThreads, kNvScoreSmem, st>>>(h->h1, 1, hd->nv_center, hd->nv_whitening, hd->nv_means, C, a->nv_base);
    if (check_launch(h, "nv_score_kernel")) return 1;
  }
  const L1Interp ig = {steps, baseline};
  for (int off = 0; off < n; off += per) {
    const int m = std::min(per, n - off);
    const uint8_t* asc = d_ascii ? d_ascii + static_cast<size_t>(off) * kWindow : h->in_stage[0];
    if (!d_ascii && launch_gather_windows(h, d_seq, d_win_start + off, d_win_len + off, m, h->in_stage[0], st)) return 1;
    if (upload_targets(a, nv->h_target + off, m, steps, st)) return 1;
    if (d_probs || nv->d_dist || nv->d_dist_target) {
      // the windows' own forward and distances: to d_dist or blockmax (scratch until the attribution step rewrites it)
      float* probs = d_probs ? probs_at(d_probs, off) : a->probs;
      float* dist = nv->d_dist ? nv->d_dist + static_cast<size_t>(off) * C : a->blockmax;
      if (forward_step(h, asc, nullptr, m, probs, nullptr, st)) return 1;
      nv_score_kernel<<<(m + kNvTile - 1) / kNvTile, kNvThreads, kNvScoreSmem, st>>>(h->h1, m, hd->nv_center, hd->nv_whitening,
                                                                                     hd->nv_means, C, dist);
      if (check_launch(h, "nv_score_kernel")) return 1;
      if (nv->d_dist_target) {
        float* out = nv->d_dist_target + static_cast<size_t>(off) * 2;
        nv_pick_kernel<<<(m + 255) / 256, 256, 0, st>>>(dist, 0, m, C, a->nv_target, steps, out);
        if (check_launch(h, "nv_pick_kernel")) return 1;
        nv_pick_kernel<<<(m + 255) / 256, 256, 0, st>>>(a->nv_base, 1, m, C, a->nv_target, steps, out + 1);
        if (check_launch(h, "nv_pick_kernel")) return 1;
      }
    }
    if (attribute_step(h, a, asc, m * steps, 0, nullptr, nullptr, st, &ig, hd, nullptr, true)) return 1;
    timer_mark(h, "ig_reduce", st);
    ig_reduce_kernel<<<dim3((kTok + 255) / 256, m), 256, 0, st>>>(a->gy1, steps, d_attr + static_cast<size_t>(off) * kTok);
    if (check_launch(h, "ig_reduce_kernel")) return 1;
    timer_mark(h, "end", st);
  }
  return 0;
}

static int attribute_ig_any(gnm_handle* h, gnm_attr* a, const char* fn, const uint8_t* d_ascii, const uint8_t* d_seq,
                            const int64_t* d_win_start, const int32_t* d_win_len, int n, int target, int steps, int baseline,
                            float* d_probs, float* d_logp, float* d_attr, void* stream, const gnm_head* hd = nullptr,
                            float* d_head_probs = nullptr, const NvAttrArgs* nv = nullptr) {
  const std::string f(fn);
  if (!h || !a) return fail(f + ": null handle or attribution context");
  if (a->h != h) return fail(f + ": the attribution context belongs to another handle");
  if (n < 0) return fail(f + ": negative window count");
  if (nv ? check_novelty(f, hd, nv, n) : check_target(f, hd, target)) return 1;
  if (steps < 1 || steps > a->max_batch)
    return fail(f + ": steps must be in [1, the attribution context's max_batch = " + std::to_string(a->max_batch) + "]");
  if (baseline != GNM_IG_BASELINE_ZERO && baseline != GNM_IG_BASELINE_N)
    return fail(f + ": baseline must be GNM_IG_BASELINE_ZERO (0) or GNM_IG_BASELINE_N (1)");
  if (h->conv_impl != 0)
    return fail(f + ": attributions need the tensor-core path (conv_impl = 0); the fp32 validation kernels have no backward pass");
  if (h->debug_stop != 0) return fail(f + ": debug_stop must be 0");
  if (n == 0) return 0;
  if (!d_attr || (!d_ascii && (!d_seq || !d_win_start || !d_win_len))) return fail(f + ": null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  if (check_device_status(h)) return 1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int per = a->max_batch / steps;                         // windows per chunk
  const int C = hd ? hd->C : 3;
  if (nv) return attribute_novelty_ig(h, a, d_ascii, d_seq, d_win_start, d_win_len, n, steps, baseline, d_probs, d_attr, st, hd,
                                      nv);
  if (d_logp) {                                                 // log p_c(x'), into column 1 of every window
    const L1Interp base = {0, baseline};
    if (forward_step(h, d_ascii ? d_ascii : h->in_stage[0], nullptr, 1, a->probs, nullptr, st, &base)) return 1;
    if (hd && head_forward_tc(h, hd, 1, a->blockmax, st)) return 1;    // the head's p(x'): blockmax, read right below
    ig_logp_kernel<<<(n + 255) / 256, 256, 0, st>>>(hd ? a->blockmax : a->probs, 1, n, attr_classes(target, C), d_logp + 1);
    if (check_launch(h, "ig_logp_kernel")) return 1;
  }
  const L1Interp ig = {steps, baseline};
  for (int off = 0; off < n; off += per) {
    const int m = std::min(per, n - off);
    const uint8_t* asc = d_ascii ? d_ascii + static_cast<size_t>(off) * kWindow : h->in_stage[0];
    if (!d_ascii && launch_gather_windows(h, d_seq, d_win_start + off, d_win_len + off, m, h->in_stage[0], st)) return 1;
    if (hd && (d_probs || d_logp || d_head_probs)) {
      // the windows' own forward and head: shipped probabilities to d_probs or the context's probs rows, the head's to
      // d_head_probs or blockmax (scratch until step 2 rewrites it), log p_c(x) from the head's
      float* probs = d_probs ? probs_at(d_probs, off) : a->probs;
      float* head_probs = d_head_probs ? d_head_probs + static_cast<size_t>(off) * C : a->blockmax;
      if (forward_step(h, asc, nullptr, m, probs, nullptr, st)) return 1;
      if (head_forward_tc(h, hd, m, head_probs, st)) return 1;
      if (d_logp) {
        ig_logp_kernel<<<(m + 255) / 256, 256, 0, st>>>(head_probs, 0, m, attr_classes(target, C),
                                                         d_logp + static_cast<size_t>(off) * 2);
        if (check_launch(h, "ig_logp_kernel")) return 1;
      }
    } else if (!hd && (d_probs || d_logp)) {
      float* probs = d_probs ? probs_at(d_probs, off) : a->blockmax;    // blockmax: scratch until step 2 rewrites it
      if (forward_step(h, asc, nullptr, m, probs, nullptr, st)) return 1;
      if (d_logp) {
        ig_logp_kernel<<<(m + 255) / 256, 256, 0, st>>>(probs, 0, m, attr_classes(target, 3),
                                                         d_logp + static_cast<size_t>(off) * 2);
        if (check_launch(h, "ig_logp_kernel")) return 1;
      }
    }
    if (attribute_step(h, a, asc, m * steps, target, nullptr, nullptr, st, &ig, hd)) return 1;
    timer_mark(h, "ig_reduce", st);
    ig_reduce_kernel<<<dim3((kTok + 255) / 256, m), 256, 0, st>>>(a->gy1, steps, d_attr + static_cast<size_t>(off) * kTok);
    if (check_launch(h, "ig_reduce_kernel")) return 1;
    timer_mark(h, "end", st);
  }
  return 0;
}

extern "C" int gnm_attribute_ig_ascii(gnm_handle* h, gnm_attr* a, const uint8_t* d_ascii, int n, int target, int steps,
                                      int baseline, float* d_probs, float* d_logp, float* d_attr, void* stream) {
  if (n > 0 && !d_ascii) return fail("gnm_attribute_ig_ascii: null buffer");
  return attribute_ig_any(h, a, "gnm_attribute_ig_ascii", d_ascii, nullptr, nullptr, nullptr, n, target, steps, baseline,
                          d_probs, d_logp, d_attr, stream);
}
extern "C" int gnm_attribute_ig_windows(gnm_handle* h, gnm_attr* a, const uint8_t* d_seq, const int64_t* d_win_start,
                                        const int32_t* d_win_len, int n, int target, int steps, int baseline, float* d_probs,
                                        float* d_logp, float* d_attr, void* stream) {
  if (n > 0 && (!d_seq || !d_win_start || !d_win_len)) return fail("gnm_attribute_ig_windows: null buffer");
  return attribute_ig_any(h, a, "gnm_attribute_ig_windows", nullptr, d_seq, d_win_start, d_win_len, n, target, steps, baseline,
                          d_probs, d_logp, d_attr, stream);
}

// ---- through a classifier head: the same passes for the head's log p_c (attribute_step); d_probs keeps the shipped classes
extern "C" int gnm_attribute_head_ascii(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_ascii, int n,
                                        int target, float* d_probs, float* d_head_probs, float* d_attr, void* stream) {
  if (!head) return fail("gnm_attribute_head_ascii: null head");
  if (n > 0 && !d_ascii) return fail("gnm_attribute_head_ascii: null buffer");
  return attribute_any(h, a, "gnm_attribute_head_ascii", d_ascii, nullptr, nullptr, nullptr, n, target, d_probs, d_attr, stream,
                       head, d_head_probs);
}
extern "C" int gnm_attribute_head_windows(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_seq,
                                          const int64_t* d_win_start, const int32_t* d_win_len, int n, int target, float* d_probs,
                                          float* d_head_probs, float* d_attr, void* stream) {
  if (!head) return fail("gnm_attribute_head_windows: null head");
  if (n > 0 && (!d_seq || !d_win_start || !d_win_len)) return fail("gnm_attribute_head_windows: null buffer");
  return attribute_any(h, a, "gnm_attribute_head_windows", nullptr, d_seq, d_win_start, d_win_len, n, target, d_probs, d_attr,
                       stream, head, d_head_probs);
}
extern "C" int gnm_attribute_head_ig_ascii(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_ascii, int n,
                                           int target, int steps, int baseline, float* d_probs, float* d_head_probs, float* d_logp,
                                           float* d_attr, void* stream) {
  if (!head) return fail("gnm_attribute_head_ig_ascii: null head");
  if (n > 0 && !d_ascii) return fail("gnm_attribute_head_ig_ascii: null buffer");
  return attribute_ig_any(h, a, "gnm_attribute_head_ig_ascii", d_ascii, nullptr, nullptr, nullptr, n, target, steps, baseline,
                          d_probs, d_logp, d_attr, stream, head, d_head_probs);
}
extern "C" int gnm_attribute_head_ig_windows(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_seq,
                                             const int64_t* d_win_start, const int32_t* d_win_len, int n, int target, int steps,
                                             int baseline, float* d_probs, float* d_head_probs, float* d_logp, float* d_attr,
                                             void* stream) {
  if (!head) return fail("gnm_attribute_head_ig_windows: null head");
  if (n > 0 && (!d_seq || !d_win_start || !d_win_len)) return fail("gnm_attribute_head_ig_windows: null buffer");
  return attribute_ig_any(h, a, "gnm_attribute_head_ig_windows", nullptr, d_seq, d_win_start, d_win_len, n, target, steps,
                          baseline, d_probs, d_logp, d_attr, stream, head, d_head_probs);
}

// ---- of a head's novelty distance to each window's target class (nv_residual_kernel, nv_grad_kernel)
extern "C" int gnm_attribute_novelty_ascii(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_ascii, int n,
                                           const int32_t* h_target, float* d_probs, float* d_dist, float* d_attr, void* stream) {
  if (!head) return fail("gnm_attribute_novelty_ascii: null head");
  if (n > 0 && !d_ascii) return fail("gnm_attribute_novelty_ascii: null buffer");
  const NvAttrArgs nv = {h_target, d_dist, nullptr};
  return attribute_any(h, a, "gnm_attribute_novelty_ascii", d_ascii, nullptr, nullptr, nullptr, n, 0, d_probs, d_attr, stream,
                       head, nullptr, &nv);
}
extern "C" int gnm_attribute_novelty_windows(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_seq,
                                             const int64_t* d_win_start, const int32_t* d_win_len, int n, const int32_t* h_target,
                                             float* d_probs, float* d_dist, float* d_attr, void* stream) {
  if (!head) return fail("gnm_attribute_novelty_windows: null head");
  if (n > 0 && (!d_seq || !d_win_start || !d_win_len)) return fail("gnm_attribute_novelty_windows: null buffer");
  const NvAttrArgs nv = {h_target, d_dist, nullptr};
  return attribute_any(h, a, "gnm_attribute_novelty_windows", nullptr, d_seq, d_win_start, d_win_len, n, 0, d_probs, d_attr,
                       stream, head, nullptr, &nv);
}
extern "C" int gnm_attribute_novelty_ig_ascii(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_ascii, int n,
                                              const int32_t* h_target, int steps, int baseline, float* d_probs, float* d_dist,
                                              float* d_dist_target, float* d_attr, void* stream) {
  if (!head) return fail("gnm_attribute_novelty_ig_ascii: null head");
  if (n > 0 && !d_ascii) return fail("gnm_attribute_novelty_ig_ascii: null buffer");
  const NvAttrArgs nv = {h_target, d_dist, d_dist_target};
  return attribute_ig_any(h, a, "gnm_attribute_novelty_ig_ascii", d_ascii, nullptr, nullptr, nullptr, n, 0, steps, baseline,
                          d_probs, nullptr, d_attr, stream, head, nullptr, &nv);
}
extern "C" int gnm_attribute_novelty_ig_windows(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_seq,
                                                const int64_t* d_win_start, const int32_t* d_win_len, int n,
                                                const int32_t* h_target, int steps, int baseline, float* d_probs, float* d_dist,
                                                float* d_dist_target, float* d_attr, void* stream) {
  if (!head) return fail("gnm_attribute_novelty_ig_windows: null head");
  if (n > 0 && (!d_seq || !d_win_start || !d_win_len)) return fail("gnm_attribute_novelty_ig_windows: null buffer");
  const NvAttrArgs nv = {h_target, d_dist, d_dist_target};
  return attribute_ig_any(h, a, "gnm_attribute_novelty_ig_windows", nullptr, d_seq, d_win_start, d_win_len, n, 0, steps,
                          baseline, d_probs, nullptr, d_attr, stream, head, nullptr, &nv);
}

extern "C" long long gnm_attr_bytes_per_window(void) {
  return static_cast<long long>(kTok) * (3 * kRowBytes + 2 * kC * 4) + 2LL * kPooled * kC * 5 +
         4LL * (256 + 2 * kLogitsLd + kPatches + kAttrPosBlocks + kUnitsPerWin * 8 + 5) +
         (8LL + 4LL) * kHidden + 4;                             // novelty attributions: r (fp64), g_h1, target
}

// ------------------------------------------------------------------------------------------------ embedding neighbours
// No handle: the search runs on the current device and the caller's stream, and its only memory is the caller's workspace.
namespace {
struct NbPlan {
  int splits = 0, tiles_per_split = 0;
  size_t q_hi = 0, q_lo = 0, r_hi = 0, r_lo = 0, p_sim = 0, p_idx = 0, bytes = 0;   // byte offsets into the workspace
};
}  // namespace

static size_t nb_align(size_t x) { return (x + 255) & ~size_t(255); }

static int nb_check_shape(const char* fn, int64_t n_query, int64_t n_ref, int k) {
  if (k < 1 || k > kNbMaxK) return fail(std::string(fn) + ": k must be in [1, 64], not " + std::to_string(k));
  if (n_query < 0 || n_ref < 0) return fail(std::string(fn) + ": negative row count");
  if (n_query > kNbRowMax || n_ref > kNbRowMax)
    return fail(std::string(fn) + ": more than 2^30 query or reference rows in one call (the kernels use 32-bit row offsets); "
                "pass the reference in chunks and merge the lists with gnm_neighbours_merge");
  return 0;
}

// Splits: enough CTAs for every SM, and at least kNbMinSplits per query tile when there are that many reference tiles.
static int nb_plan(int64_t n_query, int64_t n_ref, int k, NbPlan* pl) {
  int dev = 0, sms = 0;
  GNM_CUDA(cudaGetDevice(&dev));
  GNM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int64_t qt = (n_query + kNbBM - 1) / kNbBM, rt = (n_ref + kNbBN - 1) / kNbBN;
  NbPlan p;
  if (qt > 0 && rt > 0) {
    const int64_t want = std::max<int64_t>(kNbMinSplits, (sms + qt - 1) / qt);
    const int64_t splits = std::min<int64_t>(rt, want);
    p.tiles_per_split = static_cast<int>((rt + splits - 1) / splits);
    p.splits = static_cast<int>((rt + p.tiles_per_split - 1) / p.tiles_per_split);   // no empty split
  }
  const size_t nq = static_cast<size_t>(n_query), nr = static_cast<size_t>(n_ref);
  size_t off = 0;
  p.q_hi = off; off += nb_align(nq * kNbDim * 4);
  p.q_lo = off; off += nb_align(nq * kNbDim * 4);
  p.r_hi = off; off += nb_align(nr * kNbDim * 4);
  p.r_lo = off; off += nb_align(nr * kNbDim * 4);
  p.p_sim = off; off += nb_align(static_cast<size_t>(p.splits) * nq * k * 4);
  p.p_idx = off; off += nb_align(static_cast<size_t>(p.splits) * nq * k * 4);
  p.bytes = off;
  *pl = p;
  return 0;
}

extern "C" size_t gnm_neighbours_workspace_bytes(int64_t n_query, int64_t n_ref, int k) {
  NbPlan pl;
  if (nb_check_shape("gnm_neighbours_workspace_bytes", n_query, n_ref, k) || nb_plan(n_query, n_ref, k, &pl)) return 0;
  return pl.bytes;
}

extern "C" int gnm_embedding_neighbours(const float* d_query, int64_t n_query, const float* d_ref, int64_t n_ref,
                                        int64_t ref_index0, int64_t self_index0, int k, float* d_sim, int64_t* d_idx, void* d_work,
                                        size_t work_bytes, void* stream) {
  const char* fn = "gnm_embedding_neighbours";
  if (nb_check_shape(fn, n_query, n_ref, k)) return 1;
  if (ref_index0 < 0 || ref_index0 > INT64_MAX - n_ref) return fail(std::string(fn) + ": ref_index0 out of range");
  if (self_index0 < -1) return fail(std::string(fn) + ": self_index0 must be -1 (no self-exclusion) or >= 0");
  if (n_query == 0) return 0;
  if (!d_query || !d_sim || !d_idx || (n_ref > 0 && (!d_ref || !d_work))) return fail(std::string(fn) + ": null buffer");
  if ((reinterpret_cast<uintptr_t>(d_query) | reinterpret_cast<uintptr_t>(d_ref)) % 16)
    return fail(std::string(fn) + ": d_query and d_ref must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(d_work) % 256) return fail(std::string(fn) + ": d_work must be 256-byte aligned");
  NbPlan pl;
  if (nb_plan(n_query, n_ref, k, &pl)) return 1;
  if (n_ref > 0 && work_bytes < pl.bytes)
    return fail(std::string(fn) + ": workspace too small: " + std::to_string(work_bytes) + " bytes, " + std::to_string(pl.bytes) +
                " needed (gnm_neighbours_workspace_bytes)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nq = static_cast<int>(n_query), nr = static_cast<int>(n_ref);
  uint8_t* w = static_cast<uint8_t*>(d_work);
  float* part_sim = nullptr; int32_t* part_idx = nullptr;
  if (nr > 0) {
    float* q_hi = reinterpret_cast<float*>(w + pl.q_hi); float* q_lo = reinterpret_cast<float*>(w + pl.q_lo);
    float* r_hi = reinterpret_cast<float*>(w + pl.r_hi); float* r_lo = reinterpret_cast<float*>(w + pl.r_lo);
    part_sim = reinterpret_cast<float*>(w + pl.p_sim); part_idx = reinterpret_cast<int32_t*>(w + pl.p_idx);
    nb_prep_kernel<<<(nq + 7) / 8, 256, 0, st>>>(d_query, nq, q_hi, q_lo);
    nb_prep_kernel<<<(nr + 7) / 8, 256, 0, st>>>(d_ref, nr, r_hi, r_lo);
    GNM_CUDA(cudaGetLastError());
    PFN_encodeTiled enc = nullptr;
    if (get_encode_fn(&enc)) return 1;
    CUtensorMap tm[4];
    if (make_f32_map(enc, &tm[0], q_hi, kNbDim, nq, kNbBM) || make_f32_map(enc, &tm[1], q_lo, kNbDim, nq, kNbBM) ||
        make_f32_map(enc, &tm[2], r_hi, kNbDim, nr, kNbBN) || make_f32_map(enc, &tm[3], r_lo, kNbDim, nr, kNbBN))
      return 1;
    NbSearchParams p;
    p.part_sim = part_sim; p.part_idx = part_idx;
    p.n_query = nq; p.n_ref = nr; p.k = k; p.splits = pl.splits; p.tiles_per_split = pl.tiles_per_split;
    p.self_off = self_index0 < 0 ? LLONG_MIN : static_cast<long long>(self_index0 - ref_index0);
    p.status = nullptr;
    const int smem = nb_smem_bytes(k);
    GNM_CUDA(cudaFuncSetAttribute(nb_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    // one CTA per (query tile, split), split fastest; at most 2^23 query tiles x max(8, #SMs) splits, inside gridDim.x's 2^31 - 1
    const unsigned grid = static_cast<unsigned>(pl.splits) * static_cast<unsigned>((nq + kNbBM - 1) / kNbBM);
    nb_search_kernel<<<grid, kNbThreads, smem, st>>>(tm[0], tm[1], tm[2], tm[3], p);
    GNM_CUDA(cudaGetLastError());
  }
  nb_finalize_kernel<<<(nq + 7) / 8, 256, 0, st>>>(part_sim, part_idx, pl.splits, nq, k, static_cast<long long>(ref_index0),
                                                   d_sim, reinterpret_cast<long long*>(d_idx));
  GNM_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int gnm_neighbours_merge(float* d_sim, int64_t* d_idx, const float* d_sim_b, const int64_t* d_idx_b, int64_t n_query,
                                    int k, void* stream) {
  if (nb_check_shape("gnm_neighbours_merge", n_query, 0, k)) return 1;
  if (n_query == 0) return 0;
  if (!d_sim || !d_idx || !d_sim_b || !d_idx_b) return fail("gnm_neighbours_merge: null buffer");
  const int nq = static_cast<int>(n_query);
  nb_merge_kernel<<<(nq + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      d_sim, reinterpret_cast<long long*>(d_idx), d_sim_b, reinterpret_cast<const long long*>(d_idx_b), nq, k);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------ embedding clusters
// Workspace: the block's TF32 halves (nb_prep_kernel), then the threshold mask [n][ceil(n / 32)] words.
static size_t cl_mask_offset(int64_t n) { return 2 * nb_align(static_cast<size_t>(n) * kNbDim * 4); }
static int cl_words(int64_t n) { return static_cast<int>((n + 31) / 32); }

extern "C" size_t gnm_cluster_block_workspace_bytes(int64_t n_block) {
  if (n_block < 0 || n_block > kClMaxBlock) {
    fail("gnm_cluster_block_workspace_bytes: n_block must be in [0, " + std::to_string(kClMaxBlock) + "], not " +
         std::to_string(n_block));
    return 0;
  }
  return cl_mask_offset(n_block) + nb_align(static_cast<size_t>(n_block) * cl_words(n_block) * 4);
}

// d_probes null: every pair of the block is compared (gnm_cluster_block); else only pairs whose representative's home list is
// one of the row's probes (gnm_cluster_block_probed)
static int cluster_block_any(const char* fn, const float* d_rows, int64_t n_block, const uint8_t* d_covered, float min_similarity,
                             const int32_t* d_probes, int nprobe, const int32_t* d_home, int32_t* d_new_reps, int32_t* d_n_new,
                             void* d_work, size_t work_bytes, cudaStream_t st) {
  if (n_block < 0 || n_block > kClMaxBlock)
    return fail(std::string(fn) + ": n_block must be in [0, " + std::to_string(kClMaxBlock) + "], not " + std::to_string(n_block));
  if (!(min_similarity > 0.f && min_similarity <= 1.f))
    return fail(std::string(fn) + ": min_similarity must be in (0, 1], not " + std::to_string(min_similarity));
  if (!d_n_new || (n_block > 0 && (!d_rows || !d_covered || !d_new_reps || !d_work))) return fail(std::string(fn) + ": null buffer");
  if (reinterpret_cast<uintptr_t>(d_rows) % 16) return fail(std::string(fn) + ": d_rows must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(d_work) % 256) return fail(std::string(fn) + ": d_work must be 256-byte aligned");
  const size_t need = gnm_cluster_block_workspace_bytes(n_block);
  if (work_bytes < need)
    return fail(std::string(fn) + ": workspace too small: " + std::to_string(work_bytes) + " bytes, " + std::to_string(need) +
                " needed (gnm_cluster_block_workspace_bytes)");
  const int n = static_cast<int>(n_block), words = cl_words(n);
  uint8_t* w = static_cast<uint8_t*>(d_work);
  float* hi = reinterpret_cast<float*>(w);
  float* lo = reinterpret_cast<float*>(w + nb_align(static_cast<size_t>(n) * kNbDim * 4));
  uint32_t* mask = reinterpret_cast<uint32_t*>(w + cl_mask_offset(n));
  if (n > 0) nb_prep_kernel<<<(n + 7) / 8, 256, 0, st>>>(d_rows, n, hi, lo);
  GNM_CUDA(cudaGetLastError());
  const int rt = n > 0 ? nb_mask_tiles((n - 1) / kNbBM * kNbBM, n) : 0;     // the last query tile needs the most
  if (rt > 0) {
    PFN_encodeTiled enc = nullptr;
    if (get_encode_fn(&enc)) return 1;
    CUtensorMap tm[4];
    if (make_f32_map(enc, &tm[0], hi, kNbDim, n, kNbBM) || make_f32_map(enc, &tm[1], lo, kNbDim, n, kNbBM) ||
        make_f32_map(enc, &tm[2], hi, kNbDim, n, kNbBN) || make_f32_map(enc, &tm[3], lo, kNbDim, n, kNbBN))
      return 1;
    NbMaskParams p;
    p.mask = mask; p.n = n; p.words = words; p.tiles_per_split = kClMaskTiles; p.thr = min_similarity; p.status = nullptr;
    GNM_CUDA(cudaFuncSetAttribute(nb_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kClMaskSmem));
    dim3 grid((rt + kClMaskTiles - 1) / kClMaskTiles, (n + kNbBM - 1) / kNbBM);
    nb_mask_kernel<<<grid, kNbThreads, kClMaskSmem, st>>>(tm[0], tm[1], tm[2], tm[3], p);
    GNM_CUDA(cudaGetLastError());
    if (d_probes) {
      const long long cells = static_cast<long long>(n) * words;
      cl_probe_filter_kernel<<<static_cast<unsigned>((cells + 255) / 256), 256, 0, st>>>(mask, n, words, d_probes, nprobe, d_home);
      GNM_CUDA(cudaGetLastError());
    }
  }
  cl_resolve_kernel<<<1, kClThreads, 0, st>>>(mask, n, words, d_covered, d_new_reps, d_n_new);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int gnm_cluster_block(const float* d_rows, int64_t n_block, const uint8_t* d_covered, float min_similarity,
                                 int32_t* d_new_reps, int32_t* d_n_new, void* d_work, size_t work_bytes, void* stream) {
  return cluster_block_any("gnm_cluster_block", d_rows, n_block, d_covered, min_similarity, nullptr, 0, nullptr, d_new_reps, d_n_new,
                           d_work, work_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int gnm_cluster_block_probed(const float* d_rows, int64_t n_block, const uint8_t* d_covered, float min_similarity,
                                        const int32_t* d_probes, int nprobe, const int32_t* d_home, int32_t* d_new_reps,
                                        int32_t* d_n_new, void* d_work, size_t work_bytes, void* stream) {
  const char* fn = "gnm_cluster_block_probed";
  if (nprobe < 1 || nprobe > kIvfMaxProbe) return fail(std::string(fn) + ": nprobe must be in [1, 64], not " + std::to_string(nprobe));
  if (n_block > 0 && (!d_probes || !d_home)) return fail(std::string(fn) + ": null buffer");
  return cluster_block_any(fn, d_rows, n_block, d_covered, min_similarity, d_probes, nprobe, d_home, d_new_reps, d_n_new, d_work,
                           work_bytes, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------ window regions (regions.cuh)
// Workspace: gamma (alpha-hat during the forward pass) fp64 [W][C], then the traceback data uint32 [W] and uint16 [W].
static size_t wr_mask_offset(int64_t n, int C) { return nb_align(static_cast<size_t>(n) * C * 8); }
static size_t wr_idx_offset(int64_t n, int C) { return wr_mask_offset(n, C) + nb_align(static_cast<size_t>(n) * 4); }

extern "C" size_t gnm_window_regions_workspace_bytes(int64_t n_windows, int C) {
  if (n_windows < 0 || n_windows > INT32_MAX || C < 2 || C > kWrMaxClasses) {
    fail("gnm_window_regions_workspace_bytes: need 0 <= n_windows < 2^31 and 2 <= C <= 32, not n_windows = " +
         std::to_string(n_windows) + ", C = " + std::to_string(C));
    return 0;
  }
  return wr_idx_offset(n_windows, C) + nb_align(static_cast<size_t>(n_windows) * 2);
}

extern "C" int gnm_window_regions(const float* d_scores, int64_t n_windows, int C, const int32_t* d_offsets, int n_seqs,
                                  const int64_t* d_start, const int32_t* d_length, int stride, double mean_region_length,
                                  float* d_posterior, int32_t* d_state, uint8_t* d_region_first, int64_t* d_region_start,
                                  int64_t* d_region_end, int32_t* d_region_windows, float* d_region_posterior,
                                  float* d_region_scores, void* d_work, size_t work_bytes, void* stream) {
  const char* fn = "gnm_window_regions";
  if (C < 2 || C > kWrMaxClasses) return fail(std::string(fn) + ": C must be in [2, 32], not " + std::to_string(C));
  if (stride < 1 || stride > kWindow) return fail(std::string(fn) + ": stride must be in [1, 6000], not " + std::to_string(stride));
  if (!(mean_region_length >= 12000.0))
    return fail(std::string(fn) + ": mean_region_length must be >= 12000, not " + std::to_string(mean_region_length));
  if (n_windows < 0 || n_windows > INT32_MAX || n_seqs < 0)
    return fail(std::string(fn) + ": need 0 <= n_windows < 2^31 and n_seqs >= 0, not " + std::to_string(n_windows) + ", " +
                std::to_string(n_seqs));
  if (n_seqs == 0 || n_windows == 0) return 0;
  if (!d_offsets) return fail(std::string(fn) + ": null buffer");
  if (n_windows > 0 && (!d_scores || !d_start || !d_length || !d_posterior || !d_state || !d_region_first || !d_region_start ||
                        !d_region_end || !d_region_windows || !d_region_posterior || !d_region_scores || !d_work))
    return fail(std::string(fn) + ": null buffer");
  if (reinterpret_cast<uintptr_t>(d_work) % 256) return fail(std::string(fn) + ": d_work must be 256-byte aligned");
  const size_t need = gnm_window_regions_workspace_bytes(n_windows, C);
  if (work_bytes < need)
    return fail(std::string(fn) + ": workspace too small: " + std::to_string(work_bytes) + " bytes, " + std::to_string(need) +
                " needed (gnm_window_regions_workspace_bytes)");
  WrParams p;
  p.scores = d_scores; p.offsets = d_offsets; p.start = d_start; p.length = d_length;
  p.n_seqs = n_seqs; p.C = C; p.stride = stride;
  const double rho = stride / mean_region_length;
  p.tau = stride / 6000.0;
  p.log1p_mq = std::log1p(-rho * C / (C - 1));
  p.inv_c = 1.0 / C;
  p.log_c = std::log(static_cast<double>(C));
  p.posterior = d_posterior; p.state = d_state; p.first = d_region_first; p.r_start = d_region_start; p.r_end = d_region_end;
  p.r_windows = d_region_windows; p.r_posterior = d_region_posterior; p.r_scores = d_region_scores;
  uint8_t* w = static_cast<uint8_t*>(d_work);
  p.gam = reinterpret_cast<double*>(w);
  p.bp_mask = reinterpret_cast<uint32_t*>(w + wr_mask_offset(n_windows, C));
  p.bp_idx = reinterpret_cast<uint16_t*>(w + wr_idx_offset(n_windows, C));
  GNM_CUDA(cudaFuncSetAttribute(wr_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWrSmem));
  wr_decode_kernel<<<(n_seqs + kWrWarps - 1) / kWrWarps, kWrWarps * 32, kWrSmem, static_cast<cudaStream_t>(stream)>>>(p);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------ classifier heads (head.cuh)

extern "C" int gnm_head_destroy(gnm_head* hd) {
  if (!hd) return 0;
  for (void* p : hd->allocs) cudaFree(p);
  delete hd;
  return 0;
}

static int head_check_weights(const char* fn, const gnm_head_weights* w) {
  if (!w->dense1_kernel || !w->dense1_bias || !w->bn1.gamma || !w->bn1.beta || !w->bn1.moving_mean || !w->bn1.moving_variance ||
      !w->dense2_kernel || !w->dense2_bias)
    return fail(std::string(fn) + ": null weight pointer");
  if (w->n_classes < 2 || w->n_classes > kHeadMaxClasses)
    return fail(std::string(fn) + ": n_classes must be in [2, " + std::to_string(kHeadMaxClasses) + "], not " +
                std::to_string(w->n_classes));
  const size_t C = static_cast<size_t>(w->n_classes), H = kHidden;
  const struct { const char* name; const float* p; size_t n; } arrays[] = {
      {"dense1_kernel", w->dense1_kernel, H * H}, {"dense1_bias", w->dense1_bias, H}, {"bn1.gamma", w->bn1.gamma, H},
      {"bn1.beta", w->bn1.beta, H}, {"bn1.moving_mean", w->bn1.moving_mean, H}, {"bn1.moving_variance", w->bn1.moving_variance, H},
      {"dense2_kernel", w->dense2_kernel, H * C}, {"dense2_bias", w->dense2_bias, C}};
  for (const auto& a : arrays)
    for (size_t i = 0; i < a.n; ++i)
      if (!std::isfinite(a.p[i])) return fail(std::string(fn) + ": " + a.name + " not finite at index " + std::to_string(i));
  // fold_bn's 1 / sqrt(var + 1e-3f) is NaN or infinite unless var + 1e-3f > 0 (in fp32, as fold_bn computes it)
  for (size_t i = 0; i < H; ++i)
    if (!(w->bn1.moving_variance[i] + 1e-3f > 0.f))
      return fail(std::string(fn) + ": bn1.moving_variance + 1e-3 is not > 0 at unit " + std::to_string(i));
  return 0;
}

extern "C" int gnm_head_create(gnm_handle* h, const gnm_head_weights* w, gnm_head** out) {
  if (!h || !w || !out) return fail("gnm_head_create: null argument");
  if (head_check_weights("gnm_head_create", w)) return 1;
  GNM_CUDA(cudaSetDevice(h->device));
  gnm_head* hd = new gnm_head();
  hd->C = w->n_classes;
  *out = hd;   // so the caller can gnm_head_destroy() after a partial failure
  std::vector<float> sc, sh, thi, tlo;
  fold_bn(w->bn1, sc, sh);
  split_dense_t(w->dense1_kernel, kHidden, thi, tlo);
  if (dev_upload(hd, &hd->d1w, w->dense1_kernel, static_cast<size_t>(kHidden) * kHidden)) return 1;
  if (dev_upload(hd, &hd->d1b, w->dense1_bias, kHidden)) return 1;
  if (dev_upload(hd, &hd->scale, sc.data(), kHidden)) return 1;
  if (dev_upload(hd, &hd->shift, sh.data(), kHidden)) return 1;
  if (dev_upload(hd, &hd->dwT_hi, thi.data(), thi.size())) return 1;
  if (dev_upload(hd, &hd->dwT_lo, tlo.data(), tlo.size())) return 1;
  if (dev_upload(hd, &hd->d2w, w->dense2_kernel, static_cast<size_t>(kHidden) * hd->C)) return 1;
  if (dev_upload(hd, &hd->d2b, w->dense2_bias, hd->C)) return 1;
  PFN_encodeTiled enc = nullptr;
  if (get_encode_fn(&enc)) return 1;
  if (make_f32_map(enc, &hd->tm_b[0], hd->dwT_hi, kHidden, kHidden, kLgBN)) return 1;
  if (make_f32_map(enc, &hd->tm_b[1], hd->dwT_lo, kHidden, kHidden, kLgBN)) return 1;
  return 0;
}

// Steps of max_batch rows on the handle's head workspace (hA_hi[1] / hA_lo[1], logits_part, h2), in stream order.
extern "C" int gnm_head_forward(gnm_handle* h, const gnm_head* hd, const float* d_embed, int n, float* d_probs, void* stream) {
  if (!h || !hd) return fail("gnm_head_forward: null handle");
  if (n < 0) return fail("gnm_head_forward: negative row count");
  if (n == 0) return 0;
  if (!d_embed || !d_probs) return fail("gnm_head_forward: null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int off = 0; off < n; off += h->max_batch) {
    const int m = std::min(h->max_batch, n - off);
    const float* x = d_embed + static_cast<size_t>(off) * kHidden;
    if (h->conv_impl == 0) {
      const size_t total = static_cast<size_t>(m) * kHidden;
      head_split_tf32_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(x, h->hA_hi[1], h->hA_lo[1], total);
      if (check_launch(h, "head_split_tf32_kernel")) return 1;
      if (head_forward_tc(h, hd, m, d_probs + static_cast<size_t>(off) * hd->C, st)) return 1;
    } else {
      if (launch_sgemm(h, x, kHidden, hd->d1w, kHidden, h->h2, kHidden, m, kHidden, kHidden, hd->d1b, hd->scale, hd->shift, 1,
                       st)) return 1;
      head_softmax_kernel<<<(m * 32 + 255) / 256, 256, 0, st>>>(h->h2, hd->d2w, hd->d2b, d_probs + static_cast<size_t>(off) * hd->C,
                                                               m, hd->C);
      if (check_launch(h, "head_softmax_kernel")) return 1;
    }
  }
  return 0;
}

static int head_segment_any(gnm_handle* h, const float* d_probs, int C, const int32_t* d_offsets, int n_contigs, float* d_out,
                            void* stream, bool mean) {
  if (!h) return fail("null handle");
  if (C < 1 || C > kHeadMaxClasses) return fail("gnm_head_segment: width must be in [1, 32]");
  if (n_contigs < 0) return fail("negative contig count");
  if (n_contigs == 0) return 0;
  if (!d_probs || !d_offsets || !d_out) return fail("null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = (n_contigs + 127) / 128;
  if (mean) head_segment_reduce_kernel<true><<<grid, 128, 0, st>>>(d_probs, d_offsets, n_contigs, C, d_out);
  else head_segment_reduce_kernel<false><<<grid, 128, 0, st>>>(d_probs, d_offsets, n_contigs, C, d_out);
  return check_launch(h, "head_segment_reduce_kernel");
}
extern "C" int gnm_head_segment_mean(gnm_handle* h, const float* d_probs, int C, const int32_t* d_offsets, int n_contigs,
                                     float* d_mean, void* stream) {
  return head_segment_any(h, d_probs, C, d_offsets, n_contigs, d_mean, stream, true);
}
extern "C" int gnm_head_segment_sum(gnm_handle* h, const float* d_probs, int C, const int32_t* d_offsets, int n_contigs,
                                    float* d_sum, void* stream) {
  return head_segment_any(h, d_probs, C, d_offsets, n_contigs, d_sum, stream, false);
}

// ---- novelty (novelty.cuh)
// Workspace of gnm_novelty_fit, in this order (each part 256-byte aligned): status, class-sum partials [blocks][C][512] fp64 and
// counts [blocks][C], class means [C][512], center [512], counts [C], scatter partials [chunks][36][64][64] fp64, S, L and P
// [512][512] fp64, whitened means [C][512].
struct NvLayout {
  size_t status, part, cnt, mu, center, counts, spart, S, L, P, m, total;
  int n_blocks, n_chunks;
};
static NvLayout nv_layout(int64_t n_fit, int C) {
  NvLayout l;
  l.n_blocks = static_cast<int>((n_fit + kNvSumRows - 1) / kNvSumRows);
  l.n_chunks = static_cast<int>((n_fit + kNvChunk - 1) / kNvChunk);
  const size_t H = kHidden, c = static_cast<size_t>(C), nb = l.n_blocks, nc = l.n_chunks;
  size_t o = 0;
  l.status = o; o += nb_align(sizeof(NvStatus));
  l.part = o; o += nb_align(nb * c * H * 8);
  l.cnt = o; o += nb_align(nb * c * 8);
  l.mu = o; o += nb_align(c * H * 8);
  l.center = o; o += nb_align(H * 8);
  l.counts = o; o += nb_align(c * 8);
  l.spart = o; o += nb_align(nc * kNvTriTiles * kNvTile * kNvTile * 8);
  l.S = o; o += nb_align(H * H * 8);
  l.L = o; o += nb_align(H * H * 8);
  l.P = o; o += nb_align(H * H * 8);
  l.m = o; o += nb_align(c * H * 8);
  l.total = o;
  return l;
}

extern "C" size_t gnm_novelty_fit_workspace_bytes(int64_t n_fit, int C) {
  if (n_fit < 1 || n_fit > (int64_t(1) << 40) || C < 2 || C > kNvMaxClasses) {
    fail("gnm_novelty_fit_workspace_bytes: need 1 <= n_fit <= 2^40 and 2 <= C <= 32, not n_fit = " + std::to_string(n_fit) +
         ", C = " + std::to_string(C));
    return 0;
  }
  return nv_layout(n_fit, C).total;
}

extern "C" int gnm_novelty_fit(gnm_handle* h, const float* d_X, int64_t n_rows, const int64_t* d_idx, int64_t n_fit,
                               const int32_t* d_labels, int C, double* h_center, double* h_whitening, double* h_means,
                               double* h_min_pivot, double* h_class_means, double* h_scatter, void* d_work, size_t work_bytes,
                               void* stream) {
  const std::string fn = "gnm_novelty_fit";
  if (!h) return fail(fn + ": null handle");
  if (C < 2 || C > kNvMaxClasses) return fail(fn + ": C must be in [2, 32], not " + std::to_string(C));
  if (n_fit < 1) return fail(fn + ": no fit row");
  if (n_rows < 1) return fail(fn + ": n_rows must be >= 1");
  if (!d_X || !d_idx || !d_labels || !d_work) return fail(fn + ": null buffer");
  if (reinterpret_cast<uintptr_t>(d_work) % 256) return fail(fn + ": d_work must be 256-byte aligned");
  const size_t need = gnm_novelty_fit_workspace_bytes(n_fit, C);
  if (need == 0) return 1;
  if (work_bytes < need)
    return fail(fn + ": workspace too small: " + std::to_string(work_bytes) + " bytes, " + std::to_string(need) +
                " needed (gnm_novelty_fit_workspace_bytes)");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const NvLayout l = nv_layout(n_fit, C);
  uint8_t* w = static_cast<uint8_t*>(d_work);
  NvStatus* status = reinterpret_cast<NvStatus*>(w + l.status);
  double *part = reinterpret_cast<double*>(w + l.part), *mu = reinterpret_cast<double*>(w + l.mu);
  double *center = reinterpret_cast<double*>(w + l.center), *spart = reinterpret_cast<double*>(w + l.spart);
  double *S = reinterpret_cast<double*>(w + l.S), *L = reinterpret_cast<double*>(w + l.L), *P = reinterpret_cast<double*>(w + l.P);
  double* m = reinterpret_cast<double*>(w + l.m);
  long long *cnt = reinterpret_cast<long long*>(w + l.cnt), *counts = reinterpret_cast<long long*>(w + l.counts);
  GNM_CUDA(cudaMemsetAsync(status, 0, sizeof(NvStatus), st));
  const int sum_smem = C * kHidden * 8;
  GNM_CUDA(cudaFuncSetAttribute(nv_class_sums_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sum_smem));
  nv_class_sums_kernel<<<l.n_blocks, kHidden, sum_smem, st>>>(d_X, n_rows, d_idx, d_labels, n_fit, C, part, cnt, status);
  if (check_launch(h, "nv_class_sums_kernel")) return 1;
  nv_means_kernel<<<C + 1, kHidden, 0, st>>>(part, cnt, l.n_blocks, C, n_fit, mu, center, counts, status);
  if (check_launch(h, "nv_means_kernel")) return 1;
  nv_scatter_kernel<<<dim3(kNvTriTiles, l.n_chunks), kNvThreads, 0, st>>>(d_X, n_rows, d_idx, d_labels, n_fit, C, mu, spart, status);
  if (check_launch(h, "nv_scatter_kernel")) return 1;
  nv_scatter_reduce_kernel<<<dim3(kNvTriTiles, kNvTile * kNvTile / 256), 256, 0, st>>>(spart, l.n_chunks, n_fit, S);
  if (check_launch(h, "nv_scatter_reduce_kernel")) return 1;
  nv_factor_kernel<<<1, kNvFactorThreads, 0, st>>>(S, L, status);
  if (check_launch(h, "nv_factor_kernel")) return 1;
  nv_inverse_kernel<<<kHidden / 128, 128, 0, st>>>(L, P, status);
  if (check_launch(h, "nv_inverse_kernel")) return 1;
  nv_whiten_means_kernel<<<C, kHidden, 0, st>>>(P, mu, center, m, status);
  if (check_launch(h, "nv_whiten_means_kernel")) return 1;
  NvStatus hs;
  GNM_CUDA(cudaMemcpyAsync(&hs, status, sizeof(NvStatus), cudaMemcpyDeviceToHost, st));
  GNM_CUDA(cudaStreamSynchronize(st));
  switch (hs.code) {
    case kNvOk: break;
    case kNvBadIndex: return fail(fn + ": a fit row index is outside [0, n_rows)");
    case kNvBadLabel: return fail(fn + ": a fit row's label is outside [0, C)");
    case kNvEmptyClass: return fail(fn + ": class " + std::to_string(hs.arg) + " has no fit row");
    case kNvNoVariation: return fail(fn + ": the training windows have no within-class variation (tr S = 0)");
    case kNvNonFinite: return fail(fn + ": a fit row has a non-finite value (NaN or infinity), so tr S is not finite");
    case kNvBadPivot:
      return fail(fn + ": the shrunk covariance has a non-positive Cholesky pivot at column " + std::to_string(hs.arg));
    default: return fail(fn + ": unknown status " + std::to_string(hs.code));
  }
  const size_t H = kHidden;
  if (h_center) GNM_CUDA(cudaMemcpy(h_center, center, H * 8, cudaMemcpyDeviceToHost));
  if (h_whitening) GNM_CUDA(cudaMemcpy(h_whitening, P, H * H * 8, cudaMemcpyDeviceToHost));
  if (h_means) GNM_CUDA(cudaMemcpy(h_means, m, static_cast<size_t>(C) * H * 8, cudaMemcpyDeviceToHost));
  if (h_class_means) GNM_CUDA(cudaMemcpy(h_class_means, mu, static_cast<size_t>(C) * H * 8, cudaMemcpyDeviceToHost));
  if (h_scatter) GNM_CUDA(cudaMemcpy(h_scatter, S, H * H * 8, cudaMemcpyDeviceToHost));
  if (h_min_pivot) *h_min_pivot = hs.min_pivot;
  return 0;
}

extern "C" int gnm_head_set_novelty(gnm_handle* h, gnm_head* hd, const double* center, const double* whitening,
                                    const double* means) {
  const std::string fn = "gnm_head_set_novelty";
  if (!h || !hd) return fail(fn + ": null handle");
  if (!center || !whitening || !means) return fail(fn + ": null array");
  const size_t H = kHidden, C = static_cast<size_t>(hd->C);
  for (size_t i = 0; i < H; ++i)
    if (!std::isfinite(center[i])) return fail(fn + ": center not finite at index " + std::to_string(i));
  for (size_t i = 0; i < C * H; ++i)
    if (!std::isfinite(means[i])) return fail(fn + ": means not finite at index " + std::to_string(i));
  for (size_t i = 0; i < H; ++i)
    for (size_t j = 0; j < H; ++j) {
      const double v = whitening[i * H + j];
      if (!std::isfinite(v)) return fail(fn + ": whitening not finite at (" + std::to_string(i) + ", " + std::to_string(j) + ")");
      if (j > i && v != 0.0) return fail(fn + ": whitening is not lower triangular at (" + std::to_string(i) + ", " + std::to_string(j) + ")");
      if (j == i && !(v > 0.0)) return fail(fn + ": whitening diagonal is not positive at " + std::to_string(i));
    }
  GNM_CUDA(cudaSetDevice(h->device));
  if (!hd->nv_center) {
    if (dev_alloc(hd, &hd->nv_center, H) || dev_alloc(hd, &hd->nv_whitening, H * H) || dev_alloc(hd, &hd->nv_means, C * H)) return 1;
  }
  GNM_CUDA(cudaMemcpy(hd->nv_center, center, H * 8, cudaMemcpyHostToDevice));
  GNM_CUDA(cudaMemcpy(hd->nv_whitening, whitening, H * H * 8, cudaMemcpyHostToDevice));
  GNM_CUDA(cudaMemcpy(hd->nv_means, means, C * H * 8, cudaMemcpyHostToDevice));
  return 0;
}

extern "C" int gnm_head_novelty(gnm_handle* h, const gnm_head* hd, const float* d_embed, int n, float* d_dist, void* stream) {
  if (!h || !hd) return fail("gnm_head_novelty: null handle");
  if (!hd->nv_center) return fail("gnm_head_novelty: the head has no novelty model (gnm_head_set_novelty)");
  if (n < 0) return fail("gnm_head_novelty: negative row count");
  if (n == 0) return 0;
  if (!d_embed || !d_dist) return fail("gnm_head_novelty: null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GNM_CUDA(cudaFuncSetAttribute(nv_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kNvScoreSmem));
  nv_score_kernel<<<(n + kNvTile - 1) / kNvTile, kNvThreads, kNvScoreSmem, st>>>(d_embed, n, hd->nv_center, hd->nv_whitening,
                                                                               hd->nv_means, hd->C, d_dist);
  return check_launch(h, "nv_score_kernel");
}

// ---- training
// Flat parameter layout (gnm.h): W1 [512][512], b1, gamma, beta [512], W2 [512][C], b2 [C]; gradients, Adam m and v alike.
static size_t head_param_count(int C) { return static_cast<size_t>(kHidden) * kHidden + 3 * kHidden + static_cast<size_t>(kHidden) * C + C; }

struct gnm_head_train {
  int device = 0, C = 0, max_batch = 0, last_b = 0;
  long long launches = 0;
  uint32_t key = 0;
  long long step = 0;
  float lr = 1e-3f;
  size_t n_par = 0;
  std::vector<void*> allocs;
  float *P = nullptr, *G = nullptr, *M = nullptr, *V = nullptr, *mov_mean = nullptr, *mov_var = nullptr;
  float *Xb = nullptr, *XbT = nullptr, *z1 = nullptr, *hb = nullptr, *hT = nullptr, *logits = nullptr, *dz2 = nullptr;
  float *row_loss = nullptr, *W2T = nullptr, *dH = nullptr, *dz1 = nullptr, *stats = nullptr;
  uint8_t* mask = nullptr;
  int* bad = nullptr;                           // mapped host flag: kHeadBadIndex | kHeadBadLabel (head.cuh)
  float* par(float* base, int which) const {   // 0 W1, 1 b1, 2 gamma, 3 beta, 4 W2, 5 b2
    const size_t o[6] = {0, static_cast<size_t>(kHidden) * kHidden, static_cast<size_t>(kHidden) * kHidden + kHidden,
                         static_cast<size_t>(kHidden) * kHidden + 2 * kHidden, static_cast<size_t>(kHidden) * kHidden + 3 * kHidden,
                         static_cast<size_t>(kHidden) * kHidden + 3 * kHidden + static_cast<size_t>(kHidden) * C};
    return base + o[which];
  }
};

extern "C" int gnm_head_train_destroy(gnm_head_train* tr) {
  if (!tr) return 0;
  cudaSetDevice(tr->device);
  cudaDeviceSynchronize();
  for (void* p : tr->allocs) cudaFree(p);
  if (tr->bad) cudaFreeHost(tr->bad);
  delete tr;
  return 0;
}

extern "C" int gnm_head_train_create(int device, const gnm_head_weights* init, int max_batch, uint64_t seed, float learning_rate,
                                     gnm_head_train** out) {
  if (!init || !out) return fail("gnm_head_train_create: null argument");
  if (head_check_weights("gnm_head_train_create", init)) return 1;
  if (max_batch < 1 || max_batch > 65536) return fail("gnm_head_train_create: max_batch must be in [1, 65536]");
  if (!(learning_rate > 0.f) || !std::isfinite(learning_rate)) return fail("gnm_head_train_create: learning_rate must be > 0");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail("gnm_head_train_create: no CUDA device available");
  if (device < 0 || device >= ndev) return fail("gnm_head_train_create: bad device index");
  GNM_CUDA(cudaSetDevice(device));
  gnm_head_train* tr = new gnm_head_train();
  *out = tr;
  tr->device = device; tr->C = init->n_classes; tr->max_batch = max_batch; tr->key = head_key(seed); tr->lr = learning_rate;
  tr->n_par = head_param_count(tr->C);
  const size_t mb = static_cast<size_t>(max_batch), C = static_cast<size_t>(tr->C);
  for (float** p : {&tr->P, &tr->G, &tr->M, &tr->V})
    if (dev_alloc(tr, p, tr->n_par)) return 1;
  GNM_CUDA(cudaMemset(tr->M, 0, tr->n_par * sizeof(float)));
  GNM_CUDA(cudaMemset(tr->V, 0, tr->n_par * sizeof(float)));
  GNM_CUDA(cudaMemset(tr->G, 0, tr->n_par * sizeof(float)));
  const float* src[6] = {init->dense1_kernel, init->dense1_bias, init->bn1.gamma, init->bn1.beta, init->dense2_kernel, init->dense2_bias};
  const size_t cnt[6] = {static_cast<size_t>(kHidden) * kHidden, kHidden, kHidden, kHidden, kHidden * C, C};
  for (int i = 0; i < 6; ++i) GNM_CUDA(cudaMemcpy(tr->par(tr->P, i), src[i], cnt[i] * sizeof(float), cudaMemcpyHostToDevice));
  if (dev_upload(tr, &tr->mov_mean, init->bn1.moving_mean, kHidden)) return 1;
  if (dev_upload(tr, &tr->mov_var, init->bn1.moving_variance, kHidden)) return 1;
  for (float** p : {&tr->Xb, &tr->XbT, &tr->z1, &tr->hb, &tr->hT, &tr->dH, &tr->dz1})
    if (dev_alloc(tr, p, mb * kHidden)) return 1;
  if (dev_alloc(tr, &tr->logits, mb * C)) return 1;
  if (dev_alloc(tr, &tr->dz2, mb * C)) return 1;
  if (dev_alloc(tr, &tr->row_loss, mb)) return 1;
  if (dev_alloc(tr, &tr->W2T, kHidden * C)) return 1;
  if (dev_alloc(tr, &tr->stats, 3 * kHidden)) return 1;
  if (dev_alloc(tr, &tr->mask, mb * kHidden)) return 1;
  GNM_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&tr->bad), sizeof(int), cudaHostAllocMapped));
  *tr->bad = 0;
  return 0;
}

// Inputs an earlier step found out of range (see kHeadBadIndex); the flag is read without waiting, so a step sees the flags of
// the steps that have completed, and gnm_head_train_read, which waits, sees them all.
static int head_train_status(const gnm_head_train* tr, const char* fn) {
  const int b = *reinterpret_cast<volatile int*>(tr->bad);
  if (b & kHeadBadIndex) return fail(std::string(fn) + ": a step was given a batch index outside [0, n_rows)");
  if (b & kHeadBadLabel) return fail(std::string(fn) + ": a step was given a label outside [0, C)");
  return 0;
}

extern "C" int gnm_head_train_step(gnm_head_train* tr, const float* d_X, int64_t n_rows, const int64_t* d_idx,
                                   const int32_t* d_labels, const float* d_class_weights, int B, float* d_loss, void* stream) {
  if (!tr) return fail("gnm_head_train_step: null trainer");
  if (n_rows < 1) return fail("gnm_head_train_step: n_rows must be >= 1");
  if (head_train_status(tr, "gnm_head_train_step")) return 1;
  if (B < 1 || B > tr->max_batch) return fail("gnm_head_train_step: B must be in [1, max_batch = " + std::to_string(tr->max_batch) + "]");
  if (!d_X || !d_idx || !d_labels || !d_class_weights || !d_loss) return fail("gnm_head_train_step: null buffer");
  GNM_CUDA(cudaSetDevice(tr->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int C = tr->C;
  const size_t rows = static_cast<size_t>(B) * kHidden;
  const unsigned g_rows = static_cast<unsigned>((rows + 255) / 256);
  const int col_grid = kHidden / kHeadColBlock, col_threads = kHeadColBlock * kHeadRowGroups;
  float *W1 = tr->par(tr->P, 0), *b1 = tr->par(tr->P, 1), *gamma = tr->par(tr->P, 2), *beta = tr->par(tr->P, 3);
  float *W2 = tr->par(tr->P, 4), *b2 = tr->par(tr->P, 5);
  head_gather_kernel<<<g_rows, 256, 0, st>>>(d_X, n_rows, d_idx, B, tr->Xb, tr->XbT, tr->bad);
  if (check_launch(tr, "head_gather_kernel")) return 1;
  if (launch_sgemm(tr, tr->Xb, kHidden, W1, kHidden, tr->z1, kHidden, B, kHidden, kHidden, b1, nullptr, nullptr, 0, st)) return 1;   // z1 = x W1 + b1
  head_bn_forward_kernel<<<col_grid, col_threads, 0, st>>>(tr->z1, B, gamma, beta, tr->mov_mean, tr->mov_var, tr->key,
                                                          static_cast<uint32_t>(tr->step), tr->hb, tr->hT, tr->mask, tr->stats);
  if (check_launch(tr, "head_bn_forward_kernel")) return 1;
  if (launch_sgemm(tr, tr->hb, kHidden, W2, C, tr->logits, C, B, C, kHidden, b2, nullptr, nullptr, 0, st)) return 1;              // h W2 + b2
  head_softmax_xent_kernel<<<(B * 32 + 255) / 256, 256, 0, st>>>(tr->logits, n_rows, d_idx, d_labels, d_class_weights, B, C,
                                                                 tr->dz2, tr->row_loss, tr->bad);
  if (check_launch(tr, "head_softmax_xent_kernel")) return 1;
  head_loss_db2_kernel<<<1, 64, 0, st>>>(tr->row_loss, tr->dz2, B, C, d_loss, tr->par(tr->G, 5));
  if (check_launch(tr, "head_loss_db2_kernel")) return 1;
  if (launch_sgemm(tr, tr->hT, B, tr->dz2, C, tr->par(tr->G, 4), C, kHidden, C, B, nullptr, nullptr, nullptr, 0, st)) return 1;    // dW2 = h^T dZ2
  head_transpose_w2_kernel<<<(kHidden * C + 255) / 256, 256, 0, st>>>(W2, C, tr->W2T);
  if (check_launch(tr, "head_transpose_w2_kernel")) return 1;
  if (launch_sgemm(tr, tr->dz2, C, tr->W2T, kHidden, tr->dH, kHidden, B, kHidden, C, nullptr, nullptr, nullptr, 0, st)) return 1;  // dH = dZ2 W2^T
  head_bn_backward_kernel<<<col_grid, col_threads, 0, st>>>(tr->z1, tr->dH, tr->mask, B, gamma, beta, tr->stats, tr->dz1,
                                                           tr->par(tr->G, 1), tr->par(tr->G, 2), tr->par(tr->G, 3));
  if (check_launch(tr, "head_bn_backward_kernel")) return 1;
  if (launch_sgemm(tr, tr->XbT, B, tr->dz1, kHidden, tr->G, kHidden, kHidden, kHidden, B, nullptr, nullptr, nullptr, 0, st)) return 1;  // dW1 = x^T dZ1
  const double t = static_cast<double>(tr->step + 1);
  const float alpha = static_cast<float>(tr->lr * std::sqrt(1.0 - std::pow(0.999, t)) / (1.0 - std::pow(0.9, t)));
  head_adam_kernel<<<static_cast<unsigned>((tr->n_par + 255) / 256), 256, 0, st>>>(tr->P, tr->G, tr->M, tr->V, tr->n_par, alpha,
                                                                                    static_cast<float>(1.0 - 0.9),
                                                                                    static_cast<float>(1.0 - 0.999), 1e-7f);
  if (check_launch(tr, "head_adam_kernel")) return 1;
  tr->step++;
  tr->last_b = B;
  return 0;
}

extern "C" int gnm_head_train_read(gnm_head_train* tr, float* h_params, float* h_moving_mean, float* h_moving_variance,
                                   long long* h_step, void* stream) {
  if (!tr) return fail("gnm_head_train_read: null trainer");
  GNM_CUDA(cudaSetDevice(tr->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (h_params) GNM_CUDA(cudaMemcpyAsync(h_params, tr->P, tr->n_par * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (h_moving_mean) GNM_CUDA(cudaMemcpyAsync(h_moving_mean, tr->mov_mean, kHidden * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (h_moving_variance) GNM_CUDA(cudaMemcpyAsync(h_moving_variance, tr->mov_var, kHidden * sizeof(float), cudaMemcpyDeviceToHost, st));
  GNM_CUDA(cudaStreamSynchronize(st));
  if (h_step) *h_step = tr->step;
  return head_train_status(tr, "gnm_head_train_read");
}

extern "C" int gnm_head_train_fetch(gnm_head_train* tr, const char* which, void* h_dst, void* stream) {
  if (!tr || !which || !h_dst) return fail("gnm_head_train_fetch: null argument");
  if (!tr->last_b) return fail("gnm_head_train_fetch: no step has run on this trainer");
  GNM_CUDA(cudaSetDevice(tr->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const std::string k(which);
  const void* src = nullptr;
  size_t bytes = 0;
  if (k == "grad") { src = tr->G; bytes = tr->n_par * sizeof(float); }
  else if (k == "adam_m") { src = tr->M; bytes = tr->n_par * sizeof(float); }
  else if (k == "adam_v") { src = tr->V; bytes = tr->n_par * sizeof(float); }
  else if (k == "mask") { src = tr->mask; bytes = static_cast<size_t>(tr->last_b) * kHidden; }
  else if (k == "batch_stats") { src = tr->stats; bytes = 3 * kHidden * sizeof(float); }
  else return fail("gnm_head_train_fetch: unknown buffer " + k);
  GNM_CUDA(cudaMemcpyAsync(h_dst, src, bytes, cudaMemcpyDeviceToHost, st));
  GNM_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// ------------------------------------------------------------------------------------------------ embedding map (layout.cuh)
// No handle: the current device, the caller's stream and buffers.
static int mp_check_n(const std::string& fn, int64_t n) {
  if (n < 2 || n > kNbRowMax) return fail(fn + ": n must be in [2, 2^30], not " + std::to_string(n));
  return 0;
}

extern "C" int gnm_map_membership(const float* d_sim, const int64_t* d_idx, int64_t n, int k, double* d_mean_d, double* d_rho,
                                  double* d_sigma, double* d_w, double* d_union, void* stream) {
  const std::string fn = "gnm_map_membership";
  if (mp_check_n(fn, n)) return 1;
  if (k < 1 || k > kMpMaxK || k >= n) return fail(fn + ": k must be in [1, min(64, n - 1)], not " + std::to_string(k));
  if (!d_sim || !d_idx || !d_mean_d || !d_rho || !d_sigma || !d_w || !d_union) return fail(fn + ": null buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nn = static_cast<int>(n);
  mp_mean_kernel<<<1, kMpMeanThreads, 0, st>>>(d_sim, nn, k, d_mean_d);
  GNM_CUDA(cudaGetLastError());
  mp_sigma_kernel<<<(nn + 7) / 8, 256, 0, st>>>(d_sim, nn, k, d_mean_d, d_rho, d_sigma, d_w);
  GNM_CUDA(cudaGetLastError());
  const long long e = static_cast<long long>(n) * k;
  mp_union_kernel<<<static_cast<unsigned>((e + 255) / 256), 256, 0, st>>>(reinterpret_cast<const long long*>(d_idx), d_w, nn, k,
                                                                         d_union);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

// Workspace of gnm_map_pca, each part 256-byte aligned: the novelty fit's status, fit rows and labels, class-sum partials and
// counts, mean, count and scatter partials at C = 1.
struct MpPcaLayout {
  size_t status, idx, labels, part, cnt, mu, counts, spart, total;
  int n_blocks, n_chunks;
};
static MpPcaLayout mp_pca_layout(int64_t n) {
  MpPcaLayout l;
  l.n_blocks = static_cast<int>((n + kNvSumRows - 1) / kNvSumRows);
  l.n_chunks = static_cast<int>((n + kNvChunk - 1) / kNvChunk);
  const size_t H = kHidden, nr = static_cast<size_t>(n);
  size_t o = 0;
  l.status = o; o += nb_align(sizeof(NvStatus));
  l.idx = o; o += nb_align(nr * 8);
  l.labels = o; o += nb_align(nr * 4);
  l.part = o; o += nb_align(static_cast<size_t>(l.n_blocks) * H * 8);
  l.cnt = o; o += nb_align(static_cast<size_t>(l.n_blocks) * 8);
  l.mu = o; o += nb_align(H * 8);
  l.counts = o; o += nb_align(8);
  l.spart = o; o += nb_align(static_cast<size_t>(l.n_chunks) * kNvTriTiles * kNvTile * kNvTile * 8);
  l.total = o;
  return l;
}

extern "C" size_t gnm_map_pca_workspace_bytes(int64_t n) {
  if (mp_check_n("gnm_map_pca_workspace_bytes", n)) return 0;
  return mp_pca_layout(n).total;
}

extern "C" int gnm_map_pca(const float* d_rows, int64_t n, float* d_xhat, double* d_center, double* d_S, double* d_V, void* d_work,
                           size_t work_bytes, void* stream) {
  const std::string fn = "gnm_map_pca";
  if (mp_check_n(fn, n)) return 1;
  if (!d_rows || !d_xhat || !d_center || !d_S || !d_V || !d_work) return fail(fn + ": null buffer");
  if (reinterpret_cast<uintptr_t>(d_work) % 256) return fail(fn + ": d_work must be 256-byte aligned");
  const MpPcaLayout l = mp_pca_layout(n);
  if (work_bytes < l.total)
    return fail(fn + ": workspace too small: " + std::to_string(work_bytes) + " bytes, " + std::to_string(l.total) +
                " needed (gnm_map_pca_workspace_bytes)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nn = static_cast<int>(n);
  uint8_t* w = static_cast<uint8_t*>(d_work);
  NvStatus* status = reinterpret_cast<NvStatus*>(w + l.status);
  long long* idx = reinterpret_cast<long long*>(w + l.idx);
  int* labels = reinterpret_cast<int*>(w + l.labels);
  double *part = reinterpret_cast<double*>(w + l.part), *mu = reinterpret_cast<double*>(w + l.mu);
  double* spart = reinterpret_cast<double*>(w + l.spart);
  long long *cnt = reinterpret_cast<long long*>(w + l.cnt), *counts = reinterpret_cast<long long*>(w + l.counts);
  GNM_CUDA(cudaMemsetAsync(status, 0, sizeof(NvStatus), st));
  mp_normalize_kernel<<<(nn + 7) / 8, 256, 0, st>>>(d_rows, nn, d_xhat);
  GNM_CUDA(cudaGetLastError());
  mp_iota_kernel<<<(nn + 255) / 256, 256, 0, st>>>(nn, idx, labels);
  GNM_CUDA(cudaGetLastError());
  const int64_t* fit = reinterpret_cast<const int64_t*>(idx);
  GNM_CUDA(cudaFuncSetAttribute(nv_class_sums_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kHidden * 8));
  nv_class_sums_kernel<<<l.n_blocks, kHidden, kHidden * 8, st>>>(d_xhat, n, fit, labels, n, 1, part, cnt, status);
  GNM_CUDA(cudaGetLastError());
  nv_means_kernel<<<2, kHidden, 0, st>>>(part, cnt, l.n_blocks, 1, n, mu, d_center, counts, status);
  GNM_CUDA(cudaGetLastError());
  nv_scatter_kernel<<<dim3(kNvTriTiles, l.n_chunks), kNvThreads, 0, st>>>(d_xhat, n, fit, labels, n, 1, mu, spart, status);
  GNM_CUDA(cudaGetLastError());
  nv_scatter_reduce_kernel<<<dim3(kNvTriTiles, kNvTile * kNvTile / 256), 256, 0, st>>>(spart, l.n_chunks, n, d_S);
  GNM_CUDA(cudaGetLastError());
  mp_eig_kernel<<<1, kMpEigThreads, 0, st>>>(d_S, d_V);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

// Workspace of gnm_map_init: the projections [n][2] fp64, then max |projection| and the per-axis extent (fp64).
static size_t mp_init_ext_offset(int64_t n) { return nb_align(static_cast<size_t>(n) * 16); }

extern "C" size_t gnm_map_init_workspace_bytes(int64_t n) {
  if (mp_check_n("gnm_map_init_workspace_bytes", n)) return 0;
  return mp_init_ext_offset(n) + 256;
}

extern "C" int gnm_map_init(const float* d_xhat, int64_t n, const double* d_center, const double* d_V, uint64_t seed, float* d_Y,
                            void* d_work, size_t work_bytes, void* stream) {
  const std::string fn = "gnm_map_init";
  if (mp_check_n(fn, n)) return 1;
  if (!d_xhat || !d_center || !d_V || !d_Y || !d_work) return fail(fn + ": null buffer");
  if (reinterpret_cast<uintptr_t>(d_work) % 256) return fail(fn + ": d_work must be 256-byte aligned");
  const size_t need = gnm_map_init_workspace_bytes(n);
  if (work_bytes < need)
    return fail(fn + ": workspace too small: " + std::to_string(work_bytes) + " bytes, " + std::to_string(need) +
                " needed (gnm_map_init_workspace_bytes)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nn = static_cast<int>(n);
  uint8_t* w = static_cast<uint8_t*>(d_work);
  double* proj = reinterpret_cast<double*>(w);
  double* ext = reinterpret_cast<double*>(w + mp_init_ext_offset(n));     // [0] max |proj|; [1..4] min x, min y, max x, max y
  mp_project_kernel<<<(nn + 7) / 8, 256, 0, st>>>(d_xhat, nn, d_center, d_V, proj);
  GNM_CUDA(cudaGetLastError());
  mp_extent_kernel<<<1, 1024, 0, st>>>(proj, nullptr, 2 * static_cast<long long>(n), ext);
  GNM_CUDA(cudaGetLastError());
  const unsigned grid = static_cast<unsigned>((2 * n + 255) / 256);
  mp_noise_kernel<<<grid, 256, 0, st>>>(proj, nn, ext, head_key(seed), d_Y);
  GNM_CUDA(cudaGetLastError());
  mp_extent_kernel<<<1, 1024, 0, st>>>(nullptr, d_Y, n, ext + 1);
  GNM_CUDA(cudaGetLastError());
  mp_rescale_kernel<<<grid, 256, 0, st>>>(d_Y, nn, ext + 1);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int gnm_map_epochs(const int64_t* d_row_ptr, const int32_t* d_col, const double* d_eps, int64_t n, int epochs,
                              int e_begin, int e_end, uint64_t seed, float* d_Y, float* d_Y_tmp, void* stream) {
  const std::string fn = "gnm_map_epochs";
  if (mp_check_n(fn, n)) return 1;
  if (epochs < 1 || e_begin < 0 || e_end < e_begin || e_end > epochs)
    return fail(fn + ": need epochs >= 1 and 0 <= e_begin <= e_end <= epochs, not " + std::to_string(epochs) + ", " +
                std::to_string(e_begin) + ", " + std::to_string(e_end));
  if (!d_row_ptr || !d_col || !d_eps || !d_Y || !d_Y_tmp) return fail(fn + ": null buffer");
  if ((reinterpret_cast<uintptr_t>(d_Y) | reinterpret_cast<uintptr_t>(d_Y_tmp)) % 8)
    return fail(fn + ": d_Y and d_Y_tmp must be 8-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nn = static_cast<int>(n);
  const uint32_t key = head_key(seed);
  float2 *cur = reinterpret_cast<float2*>(d_Y), *nxt = reinterpret_cast<float2*>(d_Y_tmp);
  for (int e = std::max(e_begin, 1); e < e_end; ++e) {            // epoch 0 samples no edge
    const float alpha = static_cast<float>(1.0 - static_cast<double>(e) / epochs);
    mp_epoch_kernel<<<(nn + 7) / 8, 256, 0, st>>>(reinterpret_cast<const long long*>(d_row_ptr), d_col, d_eps, nn, e,
                                                  head_mix32(key ^ static_cast<uint32_t>(e)), alpha, cur, nxt);
    GNM_CUDA(cudaGetLastError());
    std::swap(cur, nxt);
  }
  if (cur != reinterpret_cast<float2*>(d_Y))
    GNM_CUDA(cudaMemcpyAsync(d_Y, cur, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// ------------------------------------------------------------------------------------------------ embedding index
// Centroid helpers of the spherical k-means build: the rows normalised as gnm_map_pca normalises them (mp_normalize_kernel), and
// a list's centroid as its rows' sum in row order (segment_sum_rows_kernel), normalised the same way.
extern "C" int gnm_ivf_normalize(const float* d_rows, int64_t n, float* d_out, void* stream) {
  if (n < 0 || n > kNbRowMax) return fail("gnm_ivf_normalize: n must be in [0, 2^30]");
  if (n == 0) return 0;
  if (!d_rows || !d_out) return fail("gnm_ivf_normalize: null buffer");
  const int nn = static_cast<int>(n);
  mp_normalize_kernel<<<(nn + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_rows, nn, d_out);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int gnm_ivf_centroids(const float* d_xhat, const int32_t* d_offsets, int lists, float* d_sums, float* d_centroids,
                                 void* stream) {
  if (lists < 1) return fail("gnm_ivf_centroids: lists must be >= 1, not " + std::to_string(lists));
  if (!d_xhat || !d_offsets || !d_sums || !d_centroids) return fail("gnm_ivf_centroids: null buffer");
  if ((reinterpret_cast<uintptr_t>(d_xhat) | reinterpret_cast<uintptr_t>(d_sums)) % 16)
    return fail("gnm_ivf_centroids: d_xhat and d_sums must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  segment_sum_rows_kernel<<<lists, kSegRowThreads, 0, st>>>(d_xhat, d_offsets, nullptr, d_sums);
  GNM_CUDA(cudaGetLastError());
  mp_normalize_kernel<<<(lists + 7) / 8, 256, 0, st>>>(d_sums, lists, d_centroids);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int gnm_ivf_prepare(const float* d_rows, int64_t n, float* d_hi, float* d_lo, void* stream) {
  if (n < 0 || n > kNbRowMax) return fail("gnm_ivf_prepare: n must be in [0, 2^30]");
  if (n == 0) return 0;
  if (!d_rows || !d_hi || !d_lo) return fail("gnm_ivf_prepare: null buffer");
  if ((reinterpret_cast<uintptr_t>(d_rows) | reinterpret_cast<uintptr_t>(d_hi) | reinterpret_cast<uintptr_t>(d_lo)) % 16)
    return fail("gnm_ivf_prepare: d_rows, d_hi and d_lo must be 16-byte aligned");
  const int nn = static_cast<int>(n);
  nb_prep_kernel<<<(nn + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_rows, nn, d_hi, d_lo);
  GNM_CUDA(cudaGetLastError());
  return 0;
}

namespace {
struct IvfPlan {
  long long parts = 0;                         // a bound on the partial lists: pairs x the most ranges of any list
  int bits = 1;                                // sort key bits
  size_t g_raw = 0, g_hi = 0, g_lo = 0, keys = 0, skeys = 0, vals = 0, svals = 0, slot = 0, self = 0, off = 0, pstart = 0,
         items = 0, ibase = 0, cparts = 0, pbase = 0, cub = 0, cub_bytes = 0, p_sim = 0, p_idx = 0, bytes = 0;
};
}  // namespace

static int ivf_check(const char* fn, int64_t n_pairs, int64_t n_ref, const int64_t* h_offsets, int lists, int k) {
  const std::string f(fn);
  if (k < 1 || k > kNbMaxK) return fail(f + ": k must be in [1, 64], not " + std::to_string(k));
  if (lists < 1) return fail(f + ": lists must be >= 1, not " + std::to_string(lists));
  if (n_pairs < 0 || n_pairs > kNbRowMax || n_ref < 0 || n_ref > kNbRowMax)
    return fail(f + ": need 0 <= n_pairs <= 2^30 and 0 <= n_ref <= 2^30");
  if (!h_offsets) return fail(f + ": null h_offsets");
  if (h_offsets[0] != 0 || h_offsets[lists] != n_ref) return fail(f + ": offsets must start at 0 and end at n_ref");
  for (int l = 0; l < lists; ++l)
    if (h_offsets[l + 1] < h_offsets[l]) return fail(f + ": offsets must be non-decreasing (list " + std::to_string(l) + ")");
  return 0;
}

// Every pair has at most the range count of the longest list, whatever the pairs are (duplicates included).
// grow: `off` also holds the lists' ends (gnm_ivf_search_ranges)
static int ivf_plan(int64_t n_pairs, const int64_t* h_offsets, int lists, int k, IvfPlan* pl, bool grow = false) {
  IvfPlan p;
  long long max_nr = 0;
  for (int l = 0; l < lists; ++l) max_nr = std::max(max_nr, ivf_ranges(h_offsets[l + 1] - h_offsets[l]));
  p.parts = n_pairs * max_nr;
  while ((1LL << p.bits) <= lists) ++p.bits;
  size_t sort_bytes = 0, scan_bytes = 0;
  const int np = static_cast<int>(n_pairs);
  GNM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                           static_cast<const int32_t*>(nullptr), static_cast<int32_t*>(nullptr), np, 0, p.bits));
  GNM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, static_cast<const long long*>(nullptr),
                                         static_cast<long long*>(nullptr), lists + 1));
  const size_t P = static_cast<size_t>(n_pairs), L1 = static_cast<size_t>(lists) + 1;
  size_t o = 0;
  p.g_raw = o; o += nb_align(P * kNbDim * 4);
  p.g_hi = o; o += nb_align(P * kNbDim * 4);
  p.g_lo = o; o += nb_align(P * kNbDim * 4);
  p.keys = o; o += nb_align(P * 4);
  p.skeys = o; o += nb_align(P * 4);
  p.vals = o; o += nb_align(P * 4);
  p.svals = o; o += nb_align(P * 4);
  p.slot = o; o += nb_align(P * 4);
  p.self = o; o += nb_align(P * 4);
  p.off = o; o += nb_align((grow ? L1 + lists : L1) * 8);
  p.pstart = o; o += nb_align(L1 * 4);
  p.items = o; o += nb_align(L1 * 8);
  p.ibase = o; o += nb_align(L1 * 8);
  p.cparts = o; o += nb_align(L1 * 8);
  p.pbase = o; o += nb_align(L1 * 8);
  p.cub_bytes = std::max(sort_bytes, scan_bytes);
  p.cub = o; o += nb_align(p.cub_bytes);
  p.p_sim = o; o += nb_align(static_cast<size_t>(p.parts) * k * 4);
  p.p_idx = o; o += nb_align(static_cast<size_t>(p.parts) * k * 4);
  p.bytes = o;
  *pl = p;
  return 0;
}

extern "C" size_t gnm_ivf_search_workspace_bytes(int64_t n_pairs, int64_t n_ref, const int64_t* h_offsets, int lists, int k) {
  IvfPlan pl;
  if (ivf_check("gnm_ivf_search_workspace_bytes", n_pairs, n_ref, h_offsets, lists, k) || ivf_plan(n_pairs, h_offsets, lists, k, &pl))
    return 0;
  return pl.bytes;
}

// kGrow: list l holds the rows [h_offsets[l], d_end[l]) (gnm_ivf_search_ranges), else [h_offsets[l], h_offsets[l + 1])
template <bool kGrow>
static int ivf_search_any(const char* fn, const float* d_query, int64_t n_query, const int32_t* d_pair_query,
                          const int32_t* d_pair_list, int64_t n_pairs, const float* d_ref_hi, const float* d_ref_lo, int64_t n_ref,
                          const int64_t* h_offsets, const int64_t* d_end, int lists, const int64_t* d_ref_index, int64_t self_index0,
                          int k, float* d_sim, int64_t* d_idx, void* d_work, size_t work_bytes, void* stream) {
  const std::string f(fn);
  if (ivf_check(fn, n_pairs, n_ref, h_offsets, lists, k)) return 1;
  if (n_query < 0 || n_query > kNbRowMax) return fail(f + ": n_query must be in [0, 2^30]");
  if (self_index0 < -1) return fail(f + ": self_index0 must be -1 (no self-exclusion) or >= 0");
  if (n_query == 0) return 0;
  if (!d_sim || !d_idx || (n_pairs > 0 && (!d_query || !d_pair_query || !d_pair_list || !d_work)) ||
      (n_ref > 0 && (!d_ref_hi || !d_ref_lo || !d_ref_index)) || (kGrow && n_pairs > 0 && !d_end))
    return fail(f + ": null buffer");
  if ((reinterpret_cast<uintptr_t>(d_query) | reinterpret_cast<uintptr_t>(d_ref_hi) | reinterpret_cast<uintptr_t>(d_ref_lo)) % 16)
    return fail(f + ": d_query, d_ref_hi and d_ref_lo must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(d_work) % 256) return fail(f + ": d_work must be 256-byte aligned");
  IvfPlan pl;
  if (ivf_plan(n_pairs, h_offsets, lists, k, &pl, kGrow)) return 1;
  if (n_pairs > 0 && work_bytes < pl.bytes)
    return fail(f + ": workspace too small: " + std::to_string(work_bytes) + " bytes, " + std::to_string(pl.bytes) + " needed (" + f +
                "_workspace_bytes)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nq = static_cast<int>(n_query), nr = static_cast<int>(n_ref), np = static_cast<int>(n_pairs);
  if (np == 0) {                                                  // no pair: every list padded
    ivf_merge_kernel<<<(nq + 7) / 8, 256, 0, st>>>(nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr, nq,
                                                   k, nullptr, d_sim, reinterpret_cast<long long*>(d_idx));
    GNM_CUDA(cudaGetLastError());
    return 0;
  }
  int dev = 0, sms = 0;
  GNM_CUDA(cudaGetDevice(&dev));
  GNM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  uint8_t* w = static_cast<uint8_t*>(d_work);
  auto F = [&](size_t o) { return reinterpret_cast<float*>(w + o); };
  auto U = [&](size_t o) { return reinterpret_cast<uint32_t*>(w + o); };
  auto I = [&](size_t o) { return reinterpret_cast<int32_t*>(w + o); };
  auto LL = [&](size_t o) { return reinterpret_cast<long long*>(w + o); };
  long long* off = LL(pl.off);
  GNM_CUDA(cudaMemcpyAsync(off, h_offsets, (static_cast<size_t>(lists) + 1) * 8, cudaMemcpyHostToDevice, st));
  if (kGrow) {
    ivf_ends_kernel<<<(lists + 255) / 256, 256, 0, st>>>(reinterpret_cast<const long long*>(d_end), lists, off);
    GNM_CUDA(cudaGetLastError());
  }
  ivf_keys_kernel<<<(np + 255) / 256, 256, 0, st>>>(d_pair_query, d_pair_list, np, nq, lists, U(pl.keys), I(pl.vals));
  GNM_CUDA(cudaGetLastError());
  size_t cb = pl.cub_bytes;
  GNM_CUDA(cub::DeviceRadixSort::SortPairs(w + pl.cub, cb, U(pl.keys), U(pl.skeys), I(pl.vals), I(pl.svals), np, 0, pl.bits, st));
  (kGrow ? ivf_grow_lists_kernel : ivf_lists_kernel)<<<(lists + 1 + 255) / 256, 256, 0, st>>>(U(pl.skeys), np, off, lists,
                                                                                              I(pl.pstart), LL(pl.items), LL(pl.cparts));
  GNM_CUDA(cudaGetLastError());
  cb = pl.cub_bytes;
  GNM_CUDA(cub::DeviceScan::ExclusiveSum(w + pl.cub, cb, LL(pl.items), LL(pl.ibase), lists + 1, st));
  cb = pl.cub_bytes;
  GNM_CUDA(cub::DeviceScan::ExclusiveSum(w + pl.cub, cb, LL(pl.cparts), LL(pl.pbase), lists + 1, st));
  ivf_gather_kernel<<<(np + 7) / 8, 256, 0, st>>>(d_query, d_pair_query, U(pl.skeys), I(pl.svals), np, I(pl.pstart), lists, off,
                                                  reinterpret_cast<const long long*>(d_ref_index),
                                                  static_cast<long long>(self_index0), F(pl.g_raw), I(pl.slot), I(pl.self));
  GNM_CUDA(cudaGetLastError());
  nb_prep_kernel<<<(np + 7) / 8, 256, 0, st>>>(F(pl.g_raw), np, F(pl.g_hi), F(pl.g_lo));
  GNM_CUDA(cudaGetLastError());
  if (nr > 0) {
    PFN_encodeTiled enc = nullptr;
    if (get_encode_fn(&enc)) return 1;
    CUtensorMap tm[4];
    if (make_f32_map(enc, &tm[0], F(pl.g_hi), kNbDim, np, kNbBM) || make_f32_map(enc, &tm[1], F(pl.g_lo), kNbDim, np, kNbBM) ||
        make_f32_map(enc, &tm[2], const_cast<float*>(d_ref_hi), kNbDim, nr, kNbBN) ||
        make_f32_map(enc, &tm[3], const_cast<float*>(d_ref_lo), kNbDim, nr, kNbBN))
      return 1;
    IvfSearchParams p;
    p.part_sim = F(pl.p_sim); p.part_idx = I(pl.p_idx);
    p.off = off; p.pstart = I(pl.pstart); p.ibase = LL(pl.ibase); p.pbase = LL(pl.pbase); p.self_col = I(pl.self);
    p.lists = lists; p.k = k; p.status = nullptr;
    const int smem = nb_smem_bytes(k);
    auto kernel = kGrow ? ivf_grow_search_kernel : ivf_search_kernel;
    GNM_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kernel<<<sms, kNbThreads, smem, st>>>(tm[0], tm[1], tm[2], tm[3], p);   // persistent: items round robin
    GNM_CUDA(cudaGetLastError());
  }
  if (kGrow)
    ivf_grow_merge_kernel<<<(nq + 7) / 8, 256, 0, st>>>(F(pl.p_sim), I(pl.p_idx), d_pair_query, d_pair_list, np, I(pl.slot), off, lists,
                                                        I(pl.pstart), LL(pl.pbase), nq, k,
                                                        reinterpret_cast<const long long*>(d_ref_index), d_sim,
                                                        reinterpret_cast<long long*>(d_idx));
  else
    ivf_merge_kernel<<<(nq + 7) / 8, 256, 0, st>>>(F(pl.p_sim), I(pl.p_idx), d_pair_query, d_pair_list, np, I(pl.slot), off,
                                                   I(pl.pstart), LL(pl.pbase), nq, k, reinterpret_cast<const long long*>(d_ref_index),
                                                   d_sim, reinterpret_cast<long long*>(d_idx));
  GNM_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int gnm_ivf_search(const float* d_query, int64_t n_query, const int32_t* d_pair_query, const int32_t* d_pair_list,
                              int64_t n_pairs, const float* d_ref_hi, const float* d_ref_lo, int64_t n_ref, const int64_t* h_offsets,
                              int lists, const int64_t* d_ref_index, int64_t self_index0, int k, float* d_sim, int64_t* d_idx,
                              void* d_work, size_t work_bytes, void* stream) {
  return ivf_search_any<false>("gnm_ivf_search", d_query, n_query, d_pair_query, d_pair_list, n_pairs, d_ref_hi, d_ref_lo, n_ref,
                               h_offsets, nullptr, lists, d_ref_index, self_index0, k, d_sim, d_idx, d_work, work_bytes, stream);
}

extern "C" size_t gnm_ivf_search_ranges_workspace_bytes(int64_t n_pairs, int64_t n_slots, const int64_t* h_offsets, int lists, int k) {
  IvfPlan pl;
  if (ivf_check("gnm_ivf_search_ranges_workspace_bytes", n_pairs, n_slots, h_offsets, lists, k) ||
      ivf_plan(n_pairs, h_offsets, lists, k, &pl, true))
    return 0;
  return pl.bytes;
}

extern "C" int gnm_ivf_search_ranges(const float* d_query, int64_t n_query, const int32_t* d_pair_query, const int32_t* d_pair_list,
                                     int64_t n_pairs, const float* d_slot_hi, const float* d_slot_lo, int64_t n_slots,
                                     const int64_t* h_offsets, const int64_t* d_end, int lists, const int64_t* d_slot_index, int k,
                                     float* d_sim, int64_t* d_idx, void* d_work, size_t work_bytes, void* stream) {
  return ivf_search_any<true>("gnm_ivf_search_ranges", d_query, n_query, d_pair_query, d_pair_list, n_pairs, d_slot_hi, d_slot_lo,
                              n_slots, h_offsets, d_end, lists, d_slot_index, -1, k, d_sim, d_idx, d_work, work_bytes, stream);
}
