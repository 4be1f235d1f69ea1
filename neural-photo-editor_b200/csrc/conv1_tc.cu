// conv1_tc.cu -- enc_conv1 (reference IAN_simple.py:73-83 / IAN.py:71-80: 3 -> 128 channels, 5x5, stride 2, pad 2,
// bias, LeakyRectify(0.2)) on the tensor cores.
//
// K = 3*25 = 75 is too thin for a TMA-fed tap GEMM (the input has 3 channels, not a multiple of 64), so the im2col
// tile is built by threads: 16 producer warps stage the 11 x 67 x 3 float32 input patch of a 4-row x 32-column output
// tile in shared memory, expand it to the 128 x 80 (K padded) operand, split every value into bf16 hi|lo and write it
// straight into the 128B-swizzled K-major layout wgmma reads (the same layout TMA would produce), then
// fence.proxy.async + mbarrier hand it to the consumers.  Weights (128 x 80, hi|lo) are TMA-loaded once per CTA.
// Roles: warps 0-7 two consumer warpgroups (64 operand rows each; per 64-channel half of the output 15 wgmma = 5 K-slices
// x 3 passes into main|cross register accumulators, then the epilogue = bias + LReLU + re-split), warps 8-15 im2col
// (two threads per operand row and quarter pair).
//
// Operand layout: K = 80 is one 64-wide chunk (hi plane, lo plane) plus a 16-wide tail.  The tail's hi AND lo slices share
// ONE 128-byte-row plane (hi at K-slice position 0, lo at position 1: a K = 16 slice is just a +32 B start offset in the
// descriptor), so a stage is 48 KB instead of 64 KB -- which pays for the output staging below.
//
// Output: the 128 pixels x 128 channels of a tile are 32 KB CONTIGUOUS per plane in the NHWC activation.  The epilogue
// writes the tile into four 128B-swizzled staging tiles in shared memory and one thread issues four TMA stores: whole
// lines leave the SM and no global store instruction is left in the kernel.
#include <cstdio>
#include <cstring>

#include "edge.h"
#include "tc_ptx.cuh"

namespace ian {

struct Conv1Maps {
  CUtensorMap b;   // weights: 3 blocks of [128 cout][64 k] (hi k<64 | lo k<64 | hi k 64..79, lo k 64..79, zeros)
};
struct Conv1OutMap {
  CUtensorMap out; // a1 activation [2 planes][n*1024 pixels][128 ch] bf16, box 64 ch x 128 pixels, 128B swizzle
};

namespace {

using namespace tc;

constexpr int kProducers = 256;
constexpr int kThreads = 256 + kProducers;
constexpr int kChunkPlane = 128 * 64 * 2;          // one 128-row x 64-k bf16 plane: 16 KB
constexpr int kAStage = 3 * kChunkPlane;           // k 0..63 hi | k 0..63 lo | tail plane (hi, lo slices): 48 KB
constexpr int kBBytes = 3 * kChunkPlane;           // weights, same three blocks x 128 rows: 48 KB
constexpr int kOutBytes = 4 * kChunkPlane;         // output staging: (channel half) x (hi|lo) tiles of 128 pixels x 64 ch
constexpr int kPatchRows = 11, kPatchCols = 67;    // input rows 2*p0-2 .. 2*p0+8, columns -2 .. 64
constexpr int kPatchFloats = 3 * kPatchRows * kPatchCols;
constexpr int kPatchBytes = (kPatchFloats * 4 + 15) / 16 * 16;
// no alignment slack: the kernel has no static shared memory, so the dynamic window starts 1024-aligned (the kernel traps
// if it ever does not); 227 KB per CTA minus 1 KB of margin
constexpr int kSmemBytes = 2 * kAStage + kBBytes + kOutBytes + 2 * kPatchBytes + 128 + 512;   // + barriers + staged bias
static_assert(kSmemBytes <= 232448 - 1024, "conv1_tc: shared memory budget");
constexpr int kTilesPerImage = 8;                  // 32 output rows / 4
// conv1_tangent_tc_kernel: a1 signs of this many of a thread's 32 outputs per channel half are loaded while the MMAs run,
// the rest in the epilogue; 16 or more spill at the 128-register cap of a 512-thread CTA
constexpr int kPre = 8;

// one 16-byte unit (8 consecutive k) of row m: values -> bf16 hi|lo -> swizzled position in both planes
template <int K0>
__device__ __forceinline__ void put_unit(uint8_t* stage, const float* patch, int m, int r, int c) {
  __align__(16) __nv_bfloat162 hi[4], lo[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float v[2];
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      const int k = K0 + 2 * e + d;
      if (k < 75) {
        const int ch = k / 25, i = (k % 25) / 5, j = k % 5;
        v[d] = patch[(ch * kPatchRows + 2 * r + i) * kPatchCols + 2 * c + j];
      } else {
        v[d] = 0.f;
      }
    }
    hi[e] = __floats2bfloat162_rn(v[0], v[1]);
    const float2 hf = __bfloat1622float2(hi[e]);
    lo[e] = __floats2bfloat162_rn(v[0] - hf.x, v[1] - hf.y);
  }
  constexpr int unit = (K0 % 64) / 8;
  if (K0 < 64) {
    uint8_t* base = stage + m * 128 + ((unit ^ (m & 7)) << 4);
    *reinterpret_cast<uint4*>(base) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(base + kChunkPlane) = *reinterpret_cast<const uint4*>(lo);
  } else {                                             // tail plane: hi in K-slice position 0 (units 0,1), lo in position 1 (units 2,3)
    uint8_t* row = stage + 2 * kChunkPlane + m * 128;
    *reinterpret_cast<uint4*>(row + ((unit ^ (m & 7)) << 4)) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(row + (((unit + 2) ^ (m & 7)) << 4)) = *reinterpret_cast<const uint4*>(lo);
  }
}

// the 10 sixteen-byte units (K = 80) of an operand row are split into quarters 3 | 3 | 2 | 2; a producer thread builds
// quarters q and q + 2 of its row
__device__ __forceinline__ void build_quarter(int quarter, uint8_t* stage, const float* patch, int m, int r, int c) {
  if (quarter == 0) {
    put_unit<0>(stage, patch, m, r, c); put_unit<8>(stage, patch, m, r, c); put_unit<16>(stage, patch, m, r, c);
  } else if (quarter == 1) {
    put_unit<24>(stage, patch, m, r, c); put_unit<32>(stage, patch, m, r, c); put_unit<40>(stage, patch, m, r, c);
  } else if (quarter == 2) {
    put_unit<48>(stage, patch, m, r, c); put_unit<56>(stage, patch, m, r, c);
  } else {
    put_unit<64>(stage, patch, m, r, c); put_unit<72>(stage, patch, m, r, c);
  }
}

// kTangent (conv1_tangent_tc_kernel, the encoder JVP): the same GEMM on the tangent image v, no bias, and the LeakyRectify
// derivative read from the sign of the stored forward activation a1 (hi plane, mask > 0 ? 1 : 0.2, TapGemm's ACT_MASK
// rule).  Shared memory is full, so the mask comes from global memory: kPre of a thread's 32 signs per channel half load
// while the MMAs run, the rest in the epilogue.
template <bool kTangent>
__device__ __forceinline__ void conv1_tc_body(const Conv1Maps& maps, const Conv1OutMap& omap, const float* __restrict__ x,
                                              const float* __restrict__ bias, const int n_img,
                                              const __nv_bfloat16* __restrict__ mask) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = smem_u32(smem_raw);
  if (smem_base & 1023u) __trap();                     // the 128B-swizzled tiles need 1024-byte alignment (see kSmemBytes)
  uint8_t* smem_al = smem_raw;
  const uint32_t a_base = smem_base, b_base = a_base + 2 * kAStage, o_base = b_base + kBBytes, p_base = o_base + kOutBytes;
  const uint32_t bar_base = p_base + 2 * kPatchBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (2 + s); };
  const uint32_t b_bar = bar_base + 64u;
  float* bias_s = reinterpret_cast<float*>(smem_al + (bar_base + 128u - smem_base));   // 128 floats, 16-byte aligned
  if (!kTangent && threadIdx.x < 128) bias_s[threadIdx.x] = __ldg(bias + threadIdx.x);   // the epilogue reads it for every tile

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total = n_img * kTilesPerImage;

  if (threadIdx.x == 0) {
    pdl_trigger();                                      // tapgemm.h: PDL
    for (int s = 0; s < 2; ++s) {
      mbar_init(full_bar(s), kProducers / 32);
      mbar_init(empty_bar(s), 2);                       // one arrival per consumer warpgroup
    }
    mbar_init(b_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 8) {
    // ======= consumers: wgmma per channel half, bias + LeakyRectify(0.2) + hi|lo re-split -> swizzled staging -> TMA store =======
    const int wg = warp >> 2, wtid = threadIdx.x & 127;
    const bool issuer = threadIdx.x == 0;
    if (issuer) {                                       // weights, once: three 16 KB blocks in one box (constants: no pdl_wait)
      mbar_expect_tx(b_bar, kBBytes);
      tma_load_3d(&maps.b, b_bar, b_base, 0, 0, 0);
    }
    pdl_wait();                                         // a1 may still be read by the previous step's enc_conv2 only transitively; be exact
    mbar_wait(b_bar, 0);
    uint32_t t = 0;
    for (int w = blockIdx.x; w < total; w += gridDim.x, ++t) {
      const int n = w / kTilesPerImage, p0 = (w % kTilesPerImage) * 4;
      const uint32_t s = t & 1u, use = t >> 1;
      mbar_wait(full_bar(s), use & 1u);
      const uint32_t sa = a_base + s * kAStage + wg * 64 * 128;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {                     // output channels [64h, 64h + 64)
        float am[32], ac[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) { am[j] = 0.f; ac[j] = 0.f; }
        wgmma_fence_regs(am);
        wgmma_fence_regs(ac);
        const uint32_t sb = b_base + h * 64 * 128;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 5; ++ks) {                // K = 80: slices 0..3 of the 64-wide chunk, then the tail
          const bool tail = ks == 4;
          const uint64_t ko = (uint64_t)((ks & 3) * 2);   // a K = 16 slice is 32 B = 2 descriptor address units
          const uint64_t a_hi = tail ? make_sw128_desc(sa + 2 * kChunkPlane) : make_sw128_desc(sa) + ko;
          const uint64_t a_lo = tail ? make_sw128_desc(sa + 2 * kChunkPlane) + 2 : make_sw128_desc(sa + kChunkPlane) + ko;
          const uint64_t b_hi = tail ? make_sw128_desc(sb + 2 * kChunkPlane) : make_sw128_desc(sb) + ko;
          const uint64_t b_lo = tail ? make_sw128_desc(sb + 2 * kChunkPlane) + 2 : make_sw128_desc(sb + kChunkPlane) + ko;
          const uint32_t acc = ks > 0 ? 1u : 0u;
          wgmma_bf16<64>(am, a_hi, b_hi, acc);
          wgmma_bf16<64>(ac, a_lo, b_hi, acc);
          wgmma_bf16<64>(ac, a_hi, b_lo, 1u);
        }
        wgmma_commit();
        // kTangent: the a1 signs of this thread's first kPre outputs are loaded while the MMAs run
        const __nv_bfloat16* mrow = kTangent ? mask + (long long)((n * 32 + p0) * 32 + wg * 64) * 128 + h * 64 : nullptr;
        __nv_bfloat162 mk[kTangent ? kPre / 2 : 1];
        if (kTangent) {
#pragma unroll
          for (int j = 0; j < kPre; j += 2)
            mk[kTangent ? j / 2 : 0] = *reinterpret_cast<const __nv_bfloat162*>(mrow + frag_row(wtid, j) * 128 + frag_col(wtid, j));
        }
        wgmma_wait<0>();
        wgmma_fence_regs(am);
        wgmma_fence_regs(ac);
        if (h == 1 && wtid == 0) mbar_arrive(empty_bar(s));   // this warpgroup no longer reads the operand stage
        if (h == 0 && t > 0) {                          // the previous tile's TMA stores have read the staging tiles
          if (issuer) bulk_wait_group_read0();
          asm volatile("bar.sync 1, 256;" ::: "memory");
        }
        const uint32_t o_hi = o_base + (uint32_t)(h * 2) * kChunkPlane, o_lo = o_hi + kChunkPlane;
#pragma unroll
        for (int j = 0; j < 32; j += 2) {
          const int row = wg * 64 + frag_row(wtid, j), col = frag_col(wtid, j);
          float v0, v1;
          if (kTangent) {
            const float2 m = __bfloat1622float2(j < kPre ? mk[kTangent && j < kPre ? j / 2 : 0]
                                                         : *reinterpret_cast<const __nv_bfloat162*>(mrow + row % 64 * 128 + col));
            v0 = am[j] + ac[j];
            v1 = am[j + 1] + ac[j + 1];
            v0 = m.x > 0.f ? v0 : v0 * 0.2f;
            v1 = m.y > 0.f ? v1 : v1 * 0.2f;
          } else {
            v0 = am[j] + ac[j] + bias_s[h * 64 + col];
            v1 = am[j + 1] + ac[j + 1] + bias_s[h * 64 + col + 1];
            v0 = fmaf(0.4f, fabsf(v0), 0.6f * v0);
            v1 = fmaf(0.4f, fabsf(v1), 0.6f * v1);
          }
          const __nv_bfloat162 hi = __floats2bfloat162_rn(v0, v1);
          const float2 hf = __bfloat1622float2(hi);
          const __nv_bfloat162 lo = __floats2bfloat162_rn(v0 - hf.x, v1 - hf.y);
          // channel col of the pixel's 128-byte row: 16-byte unit col/8 (128B swizzle: unit ^ row%8), 2 bytes per channel
          const uint32_t off = (uint32_t)row * 128u + ((((uint32_t)col >> 3) ^ ((uint32_t)row & 7u)) << 4) + ((uint32_t)col & 7u) * 2u;
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(o_hi + off), "r"(*reinterpret_cast<const uint32_t*>(&hi)) : "memory");
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(o_lo + off), "r"(*reinterpret_cast<const uint32_t*>(&lo)) : "memory");
        }
      }
      fence_proxy_async_smem();                          // generic-proxy writes -> visible to the TMA store
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (issuer) {
        const int pix0 = (n * 32 + p0) * 32;             // the tile's 128 pixels are consecutive in NHWC
        for (int h = 0; h < 2; ++h) {
          tma_store_3d(&omap.out, o_base + (uint32_t)(h * 2) * kChunkPlane, h * 64, pix0, 0);
          tma_store_3d(&omap.out, o_base + (uint32_t)(h * 2 + 1) * kChunkPlane, h * 64, pix0, 1);
        }
        bulk_commit_group();
      }
    }
    if (issuer) bulk_wait_group0();                      // every byte has left before the CTA retires its shared memory
  } else {
    // ===================== im2col producers (warps 8..15) =====================
    const int pt = threadIdx.x - 256;                   // 0..255
    // quarter-major: the 32 lanes of a warp build the SAME unit group of 32 consecutive rows (no divergence, and the
    // patch reads of a warp walk consecutive columns)
    const int quarter = pt >> 7, m = pt & 127;
    const int r = m >> 5, c = m & 31;
    // the patch of tile t+1 is fetched into registers while tile t is being expanded (global latency hidden)
    constexpr int kPer = (kPatchFloats + kProducers - 1) / kProducers;    // 9 floats per thread
    float pre[kPer];
    auto fetch = [&](int w) {
      const int n = w / kTilesPerImage, p0 = (w % kTilesPerImage) * 4;
#pragma unroll
      for (int e = 0; e < kPer; ++e) {
        const int i = pt + e * kProducers;
        float v = 0.f;
        if (i < kPatchFloats) {
          const int ch = i / (kPatchRows * kPatchCols), rem = i % (kPatchRows * kPatchCols);
          const int iy = 2 * p0 - 2 + rem / kPatchCols, ix = rem % kPatchCols - 2;   // rows 2*p0-2..2*p0+8, cols -2..64
          if (iy >= 0 && iy < 64 && ix >= 0 && ix < 64) v = __ldg(x + (((long long)n * 3 + ch) * 64 + iy) * 64 + ix);
        }
        pre[e] = v;
      }
    };
    pdl_wait();                                         // x may be the output of an earlier kernel of the caller's stream
    if ((int)blockIdx.x < total) fetch(blockIdx.x);
    uint32_t t = 0;
    for (int w = blockIdx.x; w < total; w += gridDim.x, ++t) {
      const uint32_t s = t & 1u, use = t >> 1;
      float* patch = reinterpret_cast<float*>(smem_al + (p_base - smem_base) + s * kPatchBytes);
      uint8_t* stage = smem_al + (a_base - smem_base) + s * kAStage;
      mbar_wait(empty_bar(s), (use & 1u) ^ 1u);         // the MMAs that read this stage have retired
#pragma unroll
      for (int e = 0; e < kPer; ++e)
        if (pt + e * kProducers < kPatchFloats) patch[pt + e * kProducers] = pre[e];
      asm volatile("bar.sync 2, 256;" ::: "memory");    // patch complete (producer warps only)
      if (w + (int)gridDim.x < total) fetch(w + gridDim.x);
      build_quarter(quarter, stage, patch, m, r, c);
      build_quarter(quarter + 2, stage, patch, m, r, c);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
      __syncwarp();
      if (lane == 0) mbar_arrive(full_bar(s));
    }
  }
}

__global__ void __launch_bounds__(kThreads, 1)
conv1_tc_kernel(const __grid_constant__ Conv1Maps maps, const __grid_constant__ Conv1OutMap omap, const float* __restrict__ x,
                const float* __restrict__ bias, const int n_img) {
  conv1_tc_body<false>(maps, omap, x, bias, n_img, nullptr);
}

// encoder JVP: v = the tangent image (n,3,64,64), omap = the tangent planes of a1, a1 = the forward activation's planes
__global__ void __launch_bounds__(kThreads, 1)
conv1_tangent_tc_kernel(const __grid_constant__ Conv1Maps maps, const __grid_constant__ Conv1OutMap omap,
                        const float* __restrict__ v, const __nv_bfloat16* __restrict__ a1, const int n_img) {
  conv1_tc_body<true>(maps, omap, v, nullptr, n_img, a1);
}

}  // namespace

Conv1Maps* conv1_build_maps(const __nv_bfloat16* wt, char* err, int errlen) {
  tc::EncodeTiledFn enc = tc::get_encode_fn();
  if (!enc) { snprintf(err, errlen, "cuTensorMapEncodeTiled entry point not available"); return nullptr; }
  Conv1Maps* m = new Conv1Maps();
  memset(m, 0, sizeof(*m));
  cuuint64_t dims[3] = {64, 128, 3};
  cuuint64_t strides[2] = {64 * 2, 128 * 64 * 2};
  cuuint32_t box[3] = {64, 128, 3};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(&m->b, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)wt, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(conv1 B) failed: %d", (int)r); delete m; return nullptr; }
  return m;
}

void conv1_free_maps(Conv1Maps* m) { delete m; }

// the a1 activation of one plan: [2 planes][n*1024 pixels][128 channels] bf16, stored in 64-channel x 128-pixel boxes
Conv1OutMap* conv1_build_out_map(__nv_bfloat16* out, long long plane, int n, char* err, int errlen) {
  tc::EncodeTiledFn enc = tc::get_encode_fn();
  if (!enc) { snprintf(err, errlen, "cuTensorMapEncodeTiled entry point not available"); return nullptr; }
  Conv1OutMap* m = new Conv1OutMap();
  memset(m, 0, sizeof(*m));
  cuuint64_t dims[3] = {128, (cuuint64_t)n * 1024, 2};
  cuuint64_t strides[2] = {128 * 2, (cuuint64_t)plane * 2};
  cuuint32_t box[3] = {64, 128, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(&m->out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)out, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(conv1 out) failed: %d", (int)r); delete m; return nullptr; }
  return m;
}

void conv1_free_out_map(Conv1OutMap* m) { delete m; }

int launch_conv1_tc(const Conv1Maps* maps, const Conv1OutMap* omap, const float* x, const float* bias, int n, cudaStream_t st) {
  static DeviceOnce attr_set;
  const int dev = cur_device();
  if (!attr_set.is_done(dev)) {
    if (cudaFuncSetAttribute(conv1_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess) return -1;
    attr_set.set_done(dev);
  }
  const int num_sms = tc_num_sms();
  const int total = n * kTilesPerImage;
  const int grid = total < num_sms ? total : num_sms;
  if (launch_pdl(conv1_tc_kernel, dim3(grid), dim3(kThreads), kSmemBytes, st, *maps, *omap, x, bias, n) != cudaSuccess) return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_conv1_tangent_tc(const Conv1Maps* maps, const Conv1OutMap* omap, const float* v, const __nv_bfloat16* a1, int n,
                            cudaStream_t st) {
  static DeviceOnce attr_set;
  const int dev = cur_device();
  if (!attr_set.is_done(dev)) {
    if (cudaFuncSetAttribute(conv1_tangent_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess) return -1;
    attr_set.set_done(dev);
  }
  const int num_sms = tc_num_sms();
  const int total = n * kTilesPerImage;
  const int grid = total < num_sms ? total : num_sms;
  if (launch_pdl(conv1_tangent_tc_kernel, dim3(grid), dim3(kThreads), kSmemBytes, st, *maps, *omap, v, a1, n) != cudaSuccess) return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ian
