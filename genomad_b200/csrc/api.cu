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
  std::vector<int32_t> band_groups[2];               // host copy: position groups per band (cost model of wv_gather_kernel's unit split)
  int32_t* cta_split = nullptr;                      // [num_sms + 1] device: unit range per CTA of the current launch
  std::vector<int32_t> split_host[2];                // host copy of the last split per IGLOO kernel (source of the async upload)
  int split_groups[2] = {-1, -1}, split_grid[2] = {-1, -1};
  float wv_cost_base = 1.f, wv_cost_group = 0.1f;    // unit cost model of wv_split: base + per position group of the busiest warp
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
  CUtensorMap tm_w[4];
  StageTimer timer;
  std::vector<void*> allocs;
};

// ------------------------------------------------------------------------------------------------
template <class T>
static int dev_upload(gnm_handle* h, T** dst, const T* src, size_t count) {
  GNM_CUDA(cudaMalloc(reinterpret_cast<void**>(dst), count * sizeof(T)));
  h->allocs.push_back(*dst);
  GNM_CUDA(cudaMemcpy(*dst, src, count * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}
template <class T>
static int dev_alloc(gnm_handle* h, T** dst, size_t count) {
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
// packed weights [stages*128 rows][128 B]; box = 128 B x 128 rows
static int make_w_map(PFN_encodeTiled enc, CUtensorMap* tm, uint8_t* base, int n_stages) {
  cuuint64_t dims[2] = {128, static_cast<cuuint64_t>(n_stages) * 128};
  cuuint64_t strides[1] = {128};
  cuuint32_t box[2] = {128, 128};
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

// One 16 KB fp16 TMA stage: B[n][kk] = fp16(part(W[k = kh*64 + kk][n]) * scale), part = hi or lo of the fp16 split.
static void pack_stage_f16(std::vector<uint8_t>& dst, const float* Wkn /* [128 k][128 n] */, int w_lo, int kh, float scale) {
  for (int n = 0; n < kC; ++n)
    for (int kk = 0; kk < 64; ++kk) {
      const float x = Wkn[static_cast<size_t>(kh * 64 + kk) * kC + n];
      const __half hi = __float2half_rn(x);
      const float v = (w_lo ? x - __half2float(hi) : __half2float(hi)) * scale;
      const uint16_t bits = __half_as_ushort(__float2half_rn(v));
      dst.push_back(static_cast<uint8_t>(bits & 0xff));
      dst.push_back(static_cast<uint8_t>(bits >> 8));
    }
}
// One 16 KB e4m3 TMA stage of the correction passes: B[n][2c + s] for the 64 input channels c of K-half kh, interleaved like the
// activation pairs (common.cuh): s = 0 multiplies lo8(A) -> e4m3(Whi * scale_hi), s = 1 multiplies hi8(A) -> e4m3(Wlo * scale_lo).
static void pack_stage_f8_pairs(std::vector<uint8_t>& dst, const float* Wkn, int kh, float scale_hi, float scale_lo) {
  for (int n = 0; n < kC; ++n)
    for (int c = 0; c < 64; ++c) {
      const float x = Wkn[static_cast<size_t>(kh * 64 + c) * kC + n];
      const float hi = __half2float(__float2half_rn(x));
      dst.push_back(static_cast<uint8_t>(__nv_cvt_float_to_fp8(hi * scale_hi, __NV_SATFINITE, __NV_E4M3)));
      dst.push_back(static_cast<uint8_t>(__nv_cvt_float_to_fp8((x - hi) * scale_lo, __NV_SATFINITE, __NV_E4M3)));
    }
}

// One IGLOO layer's patch set as the gather kernels want it (host only).
//   * fold the patch weights (Wf = w_mult * w_summer / 32, reference igloo.py:199-204 applied to rows that carry the activation
//     scale), sort the 8,400 (patch, slot) entries by position and deal them to the kGsSlots entry slots (padding slots:
//     position 0, zero weights): ent_w / ent_pos / slot_of -- patch_stream_kernel's and patch_finish*'s view;
//   * wv_gather_kernel's view of the same sorted entries: POSITION GROUPS = the entries that sit on one position, at most
//     kWgGroupMax = 4 per group (the 8 columns of the warp-level mma are 4 entries x (hi, lo); 8,400 entries hit ~4,500 positions),
//     the first group of every band of kBandRows positions, and the folded weights as that instruction's B fragments: fp16 hi / lo
//     halves of w * 2^k (k moves the largest weight to [2^13, 2^14) so that the lo halves stay in fp16's normal range; the kernel
//     multiplies the sums by unscale = 2^-k).  Fragment word order per slot: [K-half][k-step][tig] x {hi b0, hi b1, lo b0, lo b1},
//     b0 = channels (k0, k0 + 1), b1 = (k0 + 8, k0 + 9), k0 = 64 K-half + 16 k-step + 2 tig.
struct PatchPack {
  std::vector<float> ent_w;              // [kGsSlots][128]
  std::vector<int32_t> ent_pos, slot_of; // [kGsSlots], [8400]
  std::vector<int2> groups;              // {first slot, row inside the band | entries << 8}
  std::vector<int32_t> band_gstart;      // [kNumBands + 1]
  std::vector<uint32_t> frag;            // [kGsSlots][128]
  float unscale = 1.f;
};
static void pack_patches(const int32_t* patches, const float* w_mult, const float* w_summer, PatchPack& o) {
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
  float wmax = 0.f;
  for (float v : ent_w) wmax = std::max(wmax, std::fabs(v));
  int k2 = 0;
  if (wmax > 0.f && std::isfinite(wmax)) { int ex; std::frexp(wmax, &ex); k2 = std::max(-24, std::min(40, 14 - ex)); }   // wmax * 2^k2 in [2^13, 2^14)
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
  pack_patches(patches, w_mult, w_summer, pk);
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
      // common scale 2^S of the three passes (conv_t.cuh): main weights fp16(Whi * 2^d), d = 16 for |W| < 0.78
      float wmax = 0.f;
      for (size_t i = 0; i < static_cast<size_t>(kTaps) * kC * kC; ++i) wmax = std::max(wmax, std::fabs(convw[L][i]));
      if (!(wmax > 0.f) || !std::isfinite(wmax)) return fail("gnm_create: conv kernel is all-zero or not finite");
      const int shift = std::max(0, static_cast<int>(std::ceil(std::log2(wmax / 0.78f))));
      const int d = 16 - shift, S = 5 + d;
      if (d < 1) return fail("gnm_create: conv weights too large for the fp16 operand format");
      h->conv_out_scale[L] = std::ldexp(1.f, -S);
      std::vector<uint8_t> pk;                              // (region, tap): hi16.k0 x6, hi16.k1 x6, pairs.k0 x6, pairs.k1 x6
      pk.reserve(static_cast<size_t>(kConvStages) * kBStage);
      for (int kh = 0; kh < 2; ++kh)
        for (int tap = 0; tap < kTaps; ++tap)
          pack_stage_f16(pk, convw[L] + static_cast<size_t>(tap) * kC * kC, 0, kh, std::ldexp(1.f, d));
      for (int kh = 0; kh < 2; ++kh)                        // x (lo8, hi8) = (e4m3(Alo * 2^12), e4m3(Ahi * 2^7)):  (e4m3(Whi * 2^(S-12)), e4m3(Wlo * 2^(S-7)))
        for (int tap = 0; tap < kTaps; ++tap)
          pack_stage_f8_pairs(pk, convw[L] + static_cast<size_t>(tap) * kC * kC, kh, std::ldexp(1.f, S - 12), std::ldexp(1.f, S - 7));
      if (dev_upload(h, &h->wpack[L], pk.data(), pk.size())) return 1;
      if (dev_upload(h, &h->conv_w32[L], convw[L], static_cast<size_t>(kTaps) * kC * kC)) return 1;
    }
    for (int s = 0; s < 2; ++s) {                          // w_v: (K-half, weight hi/lo), unscaled fp16
      std::vector<uint8_t> pk;
      for (int kh = 0; kh < 2; ++kh)
        for (int w_lo = 0; w_lo < 2; ++w_lo) pack_stage_f16(pk, w->igloo[s].w_v, w_lo, kh, 1.f);
      if (dev_upload(h, &h->wpack[2 + s], pk.data(), pk.size())) return 1;
    }
    if (dev_upload(h, &h->conv_bias[0], w->conv2_bias, kC)) return 1;
    if (dev_upload(h, &h->conv_bias[1], w->conv3_bias, kC)) return 1;
  }
  // ---- IGLOO weights
  for (int s = 0; s < 2; ++s) {
    const gnm_igloo_weights& g = w->igloo[s];
    PatchPack pk;
    pack_patches(g.patches, g.w_mult, g.w_summer, pk);
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
      std::vector<float> sc(kHidden), sh(kHidden);
      for (int i = 0; i < kHidden; ++i) {
        const float inv = b.gamma[i] * (1.0f / std::sqrt(b.moving_variance[i] + 1e-3f));
        sc[i] = inv;
        sh[i] = b.beta[i] - b.moving_mean[i] * inv;
      }
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
      std::vector<float> thi(static_cast<size_t>(kHidden) * dk[L]), tlo(thi.size());
      for (int k = 0; k < dk[L]; ++k)
        for (int n = 0; n < kHidden; ++n)
          split_tf32(dw[L][static_cast<size_t>(k) * kHidden + n], thi[static_cast<size_t>(n) * dk[L] + k], tlo[static_cast<size_t>(n) * dk[L] + k]);
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
  if (make_w_map(enc, &h->tm_w[0], h->wpack[0], kConvStages)) return 1;
  if (make_w_map(enc, &h->tm_w[1], h->wpack[1], kConvStages)) return 1;
  if (make_w_map(enc, &h->tm_w[2], h->wpack[2], kWvStages)) return 1;
  if (make_w_map(enc, &h->tm_w[3], h->wpack[3], kWvStages)) return 1;
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
static int check_launch(gnm_handle* h, const char* what) {
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
    GNM_CUDA(cudaLaunchKernelEx(&cfg, conv_t_kernel<false>, h->tm_act[in_buf], h->tm_w[layer], p));
    return check_launch(h, "conv_t_kernel<false>(cluster)");
  }
  conv_t_kernel<false><<<grid, kConvThreads, kConvTSmem, st>>>(h->tm_act[in_buf], h->tm_w[layer], p);
  return check_launch(h, "conv_t_kernel<false>");
}
// q[s] = maxpool8(y[buf] @ w_v#s)
static int launch_wv_tc(gnm_handle* h, int s, int buf, int n, cudaStream_t st) {
  ConvTcParams p;
  p.status = h->status;
  p.experiment = 0;
  p.dbg = nullptr;
  p.bias = nullptr; p.y_out = nullptr; p.q_out = h->q[s];
  p.out_scale = 1.f / kActScale;
  p.out_fp8 = 0;
  p.n_tiles = n * kUnitsPerWin;
  const int grid = std::min(h->num_sms, p.n_tiles);
  conv_t_kernel<true><<<grid, kConvThreads, kConvTSmem, st>>>(h->tm_act[buf], h->tm_w[2 + s], p);
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
  p.q_out = h->q[s]; p.out_scale = 1.f / kActScale;
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

static int launch_sgemm(gnm_handle* h, const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N,
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
static int launch_dense_tc(gnm_handle* h, int layer, int n, float* out, float* out_hi, float* out_lo, cudaStream_t st) {
  const int K = layer == 0 ? 256 : kHidden;
  LogitsTcParams p;
  p.part = h->logits_part; p.ldc = kHidden; p.n_rows = n; p.n_cols = kHidden; p.status = h->status;
  p.chunks_total = K / kLgBK;
  p.chunks_per_split = (p.chunks_total + kHeadSplits - 1) / kHeadSplits;
  const int splits = (p.chunks_total + p.chunks_per_split - 1) / p.chunks_per_split;
  dim3 grid(kHidden / kLgBN, (n + kLgBM - 1) / kLgBM, splits);
  logits_tc_kernel<<<grid, kLgThreads, kLgSmem, st>>>(h->tm_hd_a[layer][0], h->tm_hd_a[layer][1], h->tm_hd_b[layer][0],
                                                      h->tm_hd_b[layer][1], p);
  if (check_launch(h, "logits_tc_kernel(dense)")) return 1;
  const size_t total = static_cast<size_t>(n) * kHidden;
  splitk_reduce_epi_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
      h->logits_part, out, out_hi, out_lo, n, kHidden, splits, layer == 0 ? h->d0b : h->d1b,
      layer == 0 ? h->bn0_scale : h->bn1_scale, layer == 0 ? h->bn0_shift : h->bn1_shift, 1);
  return check_launch(h, "splitk_reduce_epi_kernel");
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

// main part of a step: layer 1, the two IGLOO kernels' value projection + patch gather, conv2, conv3 (everything that streams
// the activations); returns 2 when a debug_stop cut the step short
static int forward_main(gnm_handle* h, const uint8_t* d_ascii, const uint16_t* d_tok, int n, cudaStream_t st) {
  dim3 egrid((kTok + kEmbSeg - 1) / kEmbSeg, n);
  h->ybuf_fp8lo[0] = h->ybuf_fp8lo[1] = 0;
  const bool fused = h->fuse_l1 && h->conv_impl == 0;       // layer 1 + w_v#0 in one kernel
  if (fused) {
    timer_mark(h, "layer1_wv0", st);
    FusedParams fp;
    fp.ascii = d_ascii; fp.tokens = d_tok; fp.table = h->conv1_table; fp.triple = h->conv1_triple; fp.bias = h->conv1_bias;
    fp.y_out = h->ybuf[0]; fp.q_out = h->q[0]; fp.n_units = n * kFuUnitsPerWin; fp.status = h->status;
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
// that read only q / mpi of the current buffer set and the tail-only buffers (logits, h0..h2)
static int forward_tail(gnm_handle* h, int n, float* d_probs, cudaStream_t st) {
  for (int s = 0; s < 2; ++s) {
    timer_mark(h, s ? "logits1" : "logits0", st);
    if (launch_logits(h, s, n, st)) return 1;
    timer_mark(h, s ? "attention1" : "attention0", st);
    attention_kernel<<<n, 128, 0, st>>>(h->logits, h->q[s], h->h0, h->hA_hi[0], h->hA_lo[0], s * kC);
    if (check_launch(h, "attention_kernel")) return 1;
  }
  timer_mark(h, "head", st);
  if (h->conv_impl == 0) {       // tensor cores, 3 x TF32 (the model's dense projections; the FFMA kernels stay the validation path)
    if (launch_dense_tc(h, 0, n, h->h1, h->hA_hi[1], h->hA_lo[1], st)) return 1;
    if (launch_dense_tc(h, 1, n, h->h2, nullptr, nullptr, st)) return 1;
  } else {
    if (launch_sgemm(h, h->h0, 256, h->d0w, kHidden, h->h1, kHidden, n, kHidden, 256, h->d0b, h->bn0_scale, h->bn0_shift, 1, st)) return 1;
    if (launch_sgemm(h, h->h1, kHidden, h->d1w, kHidden, h->h2, kHidden, n, kHidden, kHidden, h->d1b, h->bn1_scale, h->bn1_shift, 1, st)) return 1;
  }
  dense3_softmax_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(h->h2, h->d2w, h->d2b, d_probs, n);
  if (check_launch(h, "dense3_softmax_kernel")) return 1;
  timer_mark(h, "end", st);
  return 0;
}

// One step: n <= max_batch windows, strictly in order on one stream.
static int forward_step(gnm_handle* h, const uint8_t* d_ascii, const uint16_t* d_tok, int n, float* d_probs,
                        cudaStream_t st) {
  const int rc = forward_main(h, d_ascii, d_tok, n, st);
  if (rc) return rc == 2 ? 0 : 1;
  return forward_tail(h, n, d_probs, st);
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
  int step(const uint8_t* d_ascii, const uint16_t* d_tok, int n, float* d_probs, cudaStream_t* tail_out = nullptr) {
    if (tail_out) *tail_out = st;
    if (!on) return forward_step(h, d_ascii, d_tok, n, d_probs, st);
    const int par = steps_done & 1;
    select_set(h, par);
    if (steps_done >= 2) GNM_CUDA(cudaStreamWaitEvent(st, h->tail_done[par], 0));
    const int rc = forward_main(h, d_ascii, d_tok, n, st);
    if (rc) return 1;
    GNM_CUDA(cudaEventRecord(h->main_done[par], st));
    GNM_CUDA(cudaStreamWaitEvent(h->tail_stream, h->main_done[par], 0));
    if (forward_tail(h, n, d_probs, h->tail_stream)) return 1;
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
    const int stage = h->status->ov_stage[1] ? 1 : h->status->ov_stage[2] ? 2 : 3;       // the first layer that left the range
    h->status->act_overflow = 0;
    for (int i = 0; i < 4; ++i) h->status->ov_stage[i] = 0;
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

static int forward_any(gnm_handle* h, const uint8_t* d_ascii, const uint16_t* d_tok, int n, float* d_probs, void* stream) {
  if (!h) return fail("null handle");
  if (n < 0) return fail("negative window count");
  if (n == 0) return 0;
  if ((!d_ascii && !d_tok) || !d_probs) return fail("null buffer");
  GNM_CUDA(cudaSetDevice(h->device));
  if (check_device_status(h)) return 1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TailOverlap ov(h, st, (n + h->max_batch - 1) / h->max_batch);
  for (int off = 0; off < n; off += h->max_batch) {
    const int m = std::min(h->max_batch, n - off);
    if (ov.step(d_ascii ? d_ascii + static_cast<size_t>(off) * kWindow : nullptr,
                d_tok ? d_tok + static_cast<size_t>(off) * kTok : nullptr, m, d_probs + static_cast<size_t>(off) * 3)) return 1;
  }
  return ov.join();
}

extern "C" int gnm_forward_ascii(gnm_handle* h, const uint8_t* d_ascii, int n, float* d_probs, void* stream) {
  return forward_any(h, d_ascii, nullptr, n, d_probs, stream);
}
extern "C" int gnm_forward_tokens(gnm_handle* h, const uint16_t* d_tokens, int n, float* d_probs, void* stream) {
  return forward_any(h, nullptr, d_tokens, n, d_probs, stream);
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

// Wait for the work queued on `stream` and report device-side failures of the steps run so far (mbarrier time-outs,
// activation range overflow).  The asynchronous entry points only see such a flag on the NEXT call.
extern "C" int gnm_check_status(gnm_handle* h, void* stream) {
  if (!h) return fail("null handle");
  GNM_CUDA(cudaSetDevice(h->device));
  GNM_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  return check_device_status(h);
}

// Host buffers in, host buffers out; H2D of step i+1 overlaps compute of step i.
extern "C" int gnm_classify_host(gnm_handle* h, const uint8_t* h_ascii, int n, float* h_probs) {
  if (!h) return fail("null handle");
  if (n < 0) return fail("negative window count");
  if (n == 0) return 0;
  if (!h_ascii || !h_probs) return fail("null buffer");
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
    if (ov.step(h->in_stage[b], nullptr, m, h->out_stage[b], &tail)) return 1;
    // the input stage is only read by layer 1, but the event sits after the step's main part (the same stream); the output
    // stage of parity b is rewritten by the tail of step i+2, which is ordered after this copy on the same stream
    GNM_CUDA(cudaEventRecord(h->in_free[b], h->compute_stream));
    GNM_CUDA(cudaMemcpyAsync(h_probs + static_cast<size_t>(off) * 3, h->out_stage[b], static_cast<size_t>(m) * 3 * sizeof(float),
                             cudaMemcpyDeviceToHost, tail));
    if (ov.on) GNM_CUDA(cudaEventRecord(h->tail_done[b], tail));     // re-record: the buffer set is free once the copy is queued behind the tail
  }
  if (ov.join()) return 1;
  GNM_CUDA(cudaStreamSynchronize(h->compute_stream));
  if (ov.on) GNM_CUDA(cudaStreamSynchronize(h->tail_stream));
  return check_device_status(h);
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

extern "C" int gnm_debug_fetch(gnm_handle* h, const char* which, int n, float* d_dst, void* stream) {
  if (!h || !which || !d_dst) return fail("null argument");
  if (n < 1 || n > h->max_batch) return fail("gnm_debug_fetch: n out of range");
  GNM_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const std::string k(which);
  const float* src = nullptr;
  size_t count = 0;
  if (k == "buf0" || k == "buf1") {
    const size_t rows = static_cast<size_t>(n) * kTok;
    join_rows_kernel<<<static_cast<unsigned>((rows * kC + 255) / 256), 256, 0, st>>>(h->ybuf[k == "buf1"], d_dst, rows,
                                                                                     h->ybuf_fp8lo[k == "buf1"]);
    return check_launch(h, "join_rows_kernel");
  } else if (k == "q0" || k == "q1") { src = h->q[k == "q1"]; count = static_cast<size_t>(n) * kPooled * kC; }
  else if (k == "mpi0" || k == "mpi1") { src = h->mpi[k == "mpi1"]; count = static_cast<size_t>(n) * kPatches; }
  else if (k == "h0") { src = h->h0; count = static_cast<size_t>(n) * 256; }
  else if (k == "logits") { src = h->logits; count = static_cast<size_t>(n) * kLogitsLd; }
  else if (k == "conv_dbg") { src = reinterpret_cast<const float*>(h->conv_dbg); count = static_cast<size_t>(h->num_sms) * 16; }
  else return fail("gnm_debug_fetch: unknown buffer " + k);
  GNM_CUDA(cudaMemcpyAsync(d_dst, src, count * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}
