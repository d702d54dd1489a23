// Probe for the position-major slab of wv_gather_kernel (round 2): can a TMA tensor map list the WINDOW axis before the POSITION
// axis (strides not ascending), so that one 3-D box {128 B, 8 windows, 32 positions} lands in shared memory as
// [position][window][128 B] -- i.e. the 8 windows of one position form one 1024-byte swizzle atom, which is what ldmatrix needs
// to read "one position x 8 windows" without bank conflicts?  And does ldmatrix + mma.sync.m16n8k16 on that slab (rows 0-7 = hi16
// plane of the 8 windows, rows 8-15 = lo16 plane; B = fp16 hi / lo halves of up to 8 entries' folded weights) reproduce the patch
// gather's dot products?  Also checks the fall-back: a 2-D map (bytes of one window, windows) with one 1 KB box per position.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -o tma_probe tools/tma_order_probe.cu -lcuda && ./tma_probe
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>

constexpr int kRow = 768, kP = 70, kW = 16;       // 70 positions: the third band (64..95) is mostly out of bounds
constexpr int kRegion = 32 * 8 * 128;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__global__ void __launch_bounds__(32, 1)
probe_kernel(const __grid_constant__ CUtensorMap tm3, const __grid_constant__ CUtensorMap tm2, int mode, int band, int w0,
             uint8_t* dump /* [2][kRegion] */, const uint4* wfrag /* [8 entries][4 ks][4 tig] */, int row, int n_e,
             float* out /* [8 windows][8 entries] */) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 2 * kRegion);
  const int lane = threadIdx.x;
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(bar)));
    asm volatile("fence.mbarrier_init.release.cluster;");
  }
  __syncwarp();
  if (lane == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(2 * kRegion));
    for (int k = 0; k < 2; ++k) {                               // k = 0: hi16 channels 0..63 (row bytes 0..127), 1: lo16 (256..383)
      const int src = k * 256;
      if (mode == 0) {
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                     :: "r"(smem_u32(smem + k * kRegion)), "l"(&tm3), "r"(smem_u32(bar)), "r"(src), "r"(w0), "r"(band * 32) : "memory");
      } else {
        for (int r = 0; r < 32; ++r)                            // one 1 KB box per position; x = byte offset inside the window
          asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                       :: "r"(smem_u32(smem + k * kRegion + r * 1024)), "l"(&tm2), "r"(smem_u32(bar)),
                          "r"((band * 32 + r) * kRow + src), "r"(w0) : "memory");
      }
    }
  }
  uint32_t done = 0;
  while (!done)
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done) : "r"(smem_u32(bar)) : "memory");
  for (int i = lane; i < 2 * kRegion / 16; i += 32) reinterpret_cast<uint4*>(dump)[i] = reinterpret_cast<const uint4*>(smem)[i];

  // ---- one position group: row `row` of the band, entries 0..n_e-1, channels 0..63
  const int mat = lane >> 3, wrow = lane & 7;                    // ldmatrix: lanes 8i..8i+7 address matrix i
  const int plane = mat & 1, kchunk = mat >> 1;                  // matrices: (hi, k 0-7) (lo, k 0-7) (hi, k 8-15) (lo, k 8-15)
  const uint32_t rbase = smem_u32(smem) + plane * kRegion + row * 1024 + wrow * 128;
  const int gid = lane >> 2, tig = lane & 3;
  float acc_h[4] = {0, 0, 0, 0}, acc_l[4] = {0, 0, 0, 0};
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a0, a1, a2, a3;
    const uint32_t ad = rbase + (((ks * 2 + kchunk) ^ wrow) << 4);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(a0), "=r"(a1), "=r"(a2), "=r"(a3) : "r"(ad));
    uint4 b = make_uint4(0, 0, 0, 0);
    if (gid < n_e) b = wfrag[(gid * 4 + ks) * 4 + tig];
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(acc_h[0]), "+f"(acc_h[1]), "+f"(acc_h[2]), "+f"(acc_h[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b.x), "r"(b.y));
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(acc_l[0]), "+f"(acc_l[1]), "+f"(acc_l[2]), "+f"(acc_l[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b.z), "r"(b.w));
  }
  // rows gid (hi plane) and gid + 8 (lo plane) belong to window gid; columns 2 tig, 2 tig + 1 are entries
  out[gid * 8 + 2 * tig] = (acc_h[0] + acc_h[2]) + (acc_l[0] + acc_l[2]);
  out[gid * 8 + 2 * tig + 1] = (acc_h[1] + acc_h[3]) + (acc_l[1] + acc_l[3]);
}

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); return 2; } } while (0)

int main() {
  CK(cudaSetDevice(0));
  CK(cudaFree(0));
  std::vector<uint8_t> act(static_cast<size_t>(kW) * kP * kRow);
  std::vector<float> val(static_cast<size_t>(kW) * kP * 128);   // fp32 value hi + lo per channel
  srand(7);
  for (int w = 0; w < kW; ++w)
    for (int p = 0; p < kP; ++p) {
      uint8_t* row = &act[(static_cast<size_t>(w) * kP + p) * kRow];
      for (int i = 0; i < kRow; ++i) row[i] = static_cast<uint8_t>(rand());
      for (int c = 0; c < 128; ++c) {
        const float x = (rand() / float(RAND_MAX) - 0.5f) * 20.f;
        const __half hi = __float2half_rn(x);
        const __half lo = __float2half_rn(x - __half2float(hi));
        reinterpret_cast<__half*>(row)[c] = hi;
        reinterpret_cast<__half*>(row + 256)[c] = lo;
        val[(static_cast<size_t>(w) * kP + p) * 128 + c] = __half2float(hi) + __half2float(lo);
      }
    }
  uint8_t* d_act; CK(cudaMalloc(&d_act, act.size())); CK(cudaMemcpy(d_act, act.data(), act.size(), cudaMemcpyHostToDevice));
  CUtensorMap tm3, tm2;
  {
    cuuint64_t dims[3] = {kRow, kW, kP};
    cuuint64_t strides[2] = {static_cast<cuuint64_t>(kP) * kRow, kRow};       // window stride BEFORE the (smaller) position stride
    cuuint32_t box[3] = {128, 8, 32}, estr[3] = {1, 1, 1};
    CUresult r = cuTensorMapEncodeTiled(&tm3, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, d_act, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    printf("3-D map (bytes, window, position), strides {%d, %d}: CUresult %d\n", kP * kRow, kRow, int(r));
    if (r != CUDA_SUCCESS) memset(&tm3, 0, sizeof tm3);
    cuuint64_t dims2[2] = {static_cast<cuuint64_t>(kP) * kRow, kW};
    cuuint64_t strides2[1] = {static_cast<cuuint64_t>(kP) * kRow};
    cuuint32_t box2[2] = {128, 8}, estr2[2] = {1, 1};
    CUresult r2 = cuTensorMapEncodeTiled(&tm2, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, d_act, dims2, strides2, box2, estr2, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    printf("2-D map (bytes of a window, window): CUresult %d\n", int(r2));
    if (r != CUDA_SUCCESS && r2 != CUDA_SUCCESS) return 1;
    if (r != CUDA_SUCCESS) tm3 = tm2;
    if (r2 != CUDA_SUCCESS) tm2 = tm3;
  }
  // weights of 8 entries, channels 0..63, as mma B fragments: [entry][ks][tig] = {hi(k0,k0+1), hi(k0+8,k0+9), lo(..), lo(..)}, k0 = 16 ks + 2 tig
  std::vector<float> wgt(8 * 64);
  std::vector<uint32_t> frag(8 * 4 * 4 * 4);
  const float wscale = 4096.f;
  auto pack = [&](float x, float y) {
    return static_cast<uint32_t>(__half_as_ushort(__float2half_rn(x))) | (static_cast<uint32_t>(__half_as_ushort(__float2half_rn(y))) << 16);
  };
  for (int e = 0; e < 8; ++e) {
    for (int c = 0; c < 64; ++c) wgt[e * 64 + c] = (rand() / float(RAND_MAX) - 0.5f) * 0.02f;
    for (int ks = 0; ks < 4; ++ks)
      for (int tig = 0; tig < 4; ++tig) {
        float hi[4], lo[4];
        const int ks_k[4] = {16 * ks + 2 * tig, 16 * ks + 2 * tig + 1, 16 * ks + 2 * tig + 8, 16 * ks + 2 * tig + 9};
        for (int i = 0; i < 4; ++i) {
          const float x = wgt[e * 64 + ks_k[i]] * wscale;
          hi[i] = __half2float(__float2half_rn(x));
          lo[i] = x - hi[i];
        }
        uint32_t* f = &frag[((e * 4 + ks) * 4 + tig) * 4];
        f[0] = pack(hi[0], hi[1]); f[1] = pack(hi[2], hi[3]); f[2] = pack(lo[0], lo[1]); f[3] = pack(lo[2], lo[3]);
      }
  }
  uint4* d_frag; CK(cudaMalloc(&d_frag, frag.size() * 4)); CK(cudaMemcpy(d_frag, frag.data(), frag.size() * 4, cudaMemcpyHostToDevice));
  uint8_t* d_dump; CK(cudaMalloc(&d_dump, 2 * kRegion));
  float* d_out; CK(cudaMalloc(&d_out, 64 * 4));
  CK(cudaFuncSetAttribute(probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kRegion + 2048));
  int bad_total = 0;
  for (int mode = 0; mode < 2; ++mode)
    for (int band = 1; band < 3; ++band) {
      const int w0 = 8, row = band == 1 ? 13 : 3, n_e = 5;
      CK(cudaMemset(d_dump, 0xEE, 2 * kRegion));
      probe_kernel<<<1, 32, 2 * kRegion + 2048>>>(tm3, tm2, mode, band, w0, d_dump, d_frag, row, n_e, d_out);
      CK(cudaDeviceSynchronize());
      std::vector<uint8_t> dump(2 * kRegion);
      std::vector<float> out(64);
      CK(cudaMemcpy(dump.data(), d_dump, dump.size(), cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(out.data(), d_out, 256, cudaMemcpyDeviceToHost));
      int bad = 0;
      for (int k = 0; k < 2; ++k)
        for (int r = 0; r < 32; ++r)
          for (int w = 0; w < 8; ++w)
            for (int ch = 0; ch < 8; ++ch)
              for (int b = 0; b < 16; ++b) {
                const int p = band * 32 + r;
                const uint8_t want = p < kP ? act[(static_cast<size_t>(w0 + w) * kP + p) * kRow + k * 256 + ch * 16 + b] : 0;
                const uint8_t got = dump[k * kRegion + r * 1024 + w * 128 + ((ch ^ w) << 4) + b];
                bad += want != got;
              }
      double maxerr = 0, maxref = 0;
      for (int w = 0; w < 8; ++w)
        for (int e = 0; e < 8; ++e) {
          double ref = 0;
          const int p = band * 32 + row;
          if (e < n_e && p < kP)
            for (int c = 0; c < 64; ++c) ref += double(val[(static_cast<size_t>(w0 + w) * kP + p) * 128 + c]) * double(wgt[e * 64 + c]);
          const double got = out[w * 8 + e] / wscale;
          maxerr = fmax(maxerr, fabs(got - ref));
          maxref = fmax(maxref, fabs(ref));
        }
      printf("mode %d (%s) band %d: slab image mismatches %d of %d bytes; gather max |err| %.3e (max |ref| %.3e)\n", mode,
             mode == 0 ? "one 3-D box per region" : "32 2-D boxes per region", band, bad, 2 * kRegion, maxerr, maxref);
      bad_total += bad + (maxerr > 1e-5 * fmax(maxref, 1.0));
    }
  printf(bad_total ? "PROBE FAILED\n" : "PROBE OK\n");
  return bad_total ? 1 : 0;
}
