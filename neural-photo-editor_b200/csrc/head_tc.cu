// head_tc.cu -- the RGB-Beta head of IAN.py / IANv1.py (reference IAN.py:183-207, layers.py:207-258, 397-408) without the
// HBM tap table.
//
// The head applies three 128 -> 2 channel MDC convolutions (scales [2,3,4]: 33 distinct dilated tap offsets, halo 4) to
// the 64x64x128 feature map, then an autoregressive 2->2 / 4->2 channel pair of MDC convolutions with sigmoids and the
// Beta mean 2a/(a+b)-1.  Round 1 ran the first part as a dense 128 -> 33*6 GEMM into a channel-major table in HBM
// (3.2 MB per image) that a gather kernel read back: ~6x the algorithmic bytes, 0.56 + 0.26 ms at batch 512.
//
// head_tc_kernel: a work item is (image, conv k in {R, G_a, B_a}).  The CTA streams the image's 32 M tiles (2 rows x 64
// pixels) through ONE dense GEMM each,  T[pixel][t*2+f] = sum_c h[pixel][c] * Wk[t][f][c]  (N = 66 -> 80, K = 128: no
// shifts, the feature map is staged exactly once per conv), drains T to shared memory, and every epilogue thread adds
// the taps that land on ITS 16 output pixels,  ha[p][f] += T[p + off_t][t*2+f],  into registers (weight rows are sorted by
// the taps' row offset; the [2,3,4]-scale tap set is analytic, so the gather needs no table).  No atomics, fixed order.
// Roles: warp 16 TMA (weights per item, A ring); warps 0-15 four consumer warpgroups, one per (64-row half, 40-column
// half) of the tile's 128 x 80 result (float32 = 3-pass bf16 split into main|cross register accumulators, or single
// pass), which then drain their fragments into the shared T tile and run the gather.
// The autoregressive part (sigmoid R; G from 33 taps of R; B from 33 taps of [R,G]; Beta means) stays the three per-pixel
// kernels of edge_kernels.cu, reading this kernel's planar output: a one-CTA-per-image version with R and G in shared
// memory was tried and measured 3x slower (512 CTAs of dependent shared-memory chains vs 2 M independent threads on L2).
#include <cstdio>
#include <cstring>

#include "edge.h"
#include "tc_ptx.cuh"

namespace ian {

struct HeadMaps {
  CUtensorMap a, a1;   // feature map planes (C=128, W=64, H=64, N, planes): box {64 ch, 64, 2, 1, planes}
  CUtensorMap b, b1;   // weights (K=128, 3*80 rows, planes): box {64, 80, planes}
};

namespace {

using namespace tc;

constexpr int kEpiThreads = 512;              // 16 consumer warps: the drain + gather is latency-bound, more warps hide it
constexpr int kThreads = 32 + kEpiThreads;
constexpr int BN = 80;                        // 33 taps x 2 filters = 66, padded to a multiple of 16
constexpr int kNT = 33;
constexpr int kTLd = 67;                      // T row pitch in floats (odd: conflict-free column access)
constexpr int kTBytes = 128 * kTLd * 4;
constexpr int kTilesPerImage = 32;

template <int PASSES> struct HeadCfg {
  // the A ring is what hides the TMA round trip: a tile is only two K chunks, so its depth in TILES is kAStages / 2.  The
  // ring takes the shared memory left: 4 stages of 32 KB in float32 mode, 8 of 16 KB in bf16 mode.
  static constexpr int kAStages = PASSES == 3 ? 4 : 8;
  static constexpr int kPlanes = PASSES == 3 ? 2 : 1;
  static constexpr int kAStage = 128 * 64 * 2 * kPlanes;      // one K chunk of an A tile
  static constexpr int kBChunk = BN * 64 * 2 * kPlanes;       // one K chunk of the conv's weights
  static constexpr int kSmemBytes = 1024 + kAStages * kAStage + 2 * kBChunk + kTBytes + 256;
};

template <int PASSES>
__global__ void __launch_bounds__(kThreads, 1)
head_tc_kernel(const __grid_constant__ HeadMaps maps, float* __restrict__ ha /*[n][6][4096]*/, const int n_img) {
  using Cfg = HeadCfg<PASSES>;
  constexpr int kAStages = Cfg::kAStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t a_base = smem_base;
  const uint32_t b_base = a_base + kAStages * Cfg::kAStage;
  const uint32_t t_base = b_base + 2 * Cfg::kBChunk;
  const uint32_t bar_base = t_base + kTBytes;
  float* Ts = reinterpret_cast<float*>(smem_al + (t_base - smem_base));
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kAStages + s); };
  const uint32_t bfull_bar = bar_base + 8u * (2 * kAStages);
  const uint32_t bempty_bar = bar_base + 8u * (2 * kAStages + 1);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total = n_img * 3;

  if (threadIdx.x == 0) {
    pdl_trigger();                                      // tapgemm.h: PDL
    for (int s = 0; s < kAStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 4); }
    mbar_init(bfull_bar, 1);
    mbar_init(bempty_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                                           // prologue done; the feature map / ha below belong to the chain

  if (warp == kEpiThreads / 32) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      uint32_t i = 0, it = 0;
      for (int w = blockIdx.x; w < total; w += gridDim.x, ++it) {
        const int n = w / 3, k = w % 3;
        mbar_wait(bempty_bar, (it & 1u) ^ 1u);           // the previous item's MMAs have finished reading the weights
        mbar_expect_tx(bfull_bar, 2 * Cfg::kBChunk);
        tma_load_3d(PASSES == 3 ? &maps.b : &maps.b1, bfull_bar, b_base, 0, k * BN, 0);
        tma_load_3d(PASSES == 3 ? &maps.b : &maps.b1, bfull_bar, b_base + Cfg::kBChunk, 64, k * BN, 0);
        for (int mt = 0; mt < kTilesPerImage; ++mt)
          for (int c = 0; c < 2; ++c, ++i) {
            const int s = i % kAStages;
            mbar_wait(empty_bar(s), ((i / kAStages) & 1u) ^ 1u);
            mbar_expect_tx(full_bar(s), Cfg::kAStage);
            tma_load_5d(PASSES == 3 ? &maps.a : &maps.a1, full_bar(s), a_base + s * Cfg::kAStage, c * 64, 0, 2 * mt, n, 0);
          }
      }
    }
    return;
  }
  // ===================== consumers: wgmma -> smem T tile -> tap gather into registers =====================
  constexpr int NW = BN / 2;                            // columns of one warpgroup's accumulator
  const int et = threadIdx.x;                           // 0..511
  const int wg = warp >> 2, wtid = threadIdx.x & 127;
  const int row0 = (wg & 1) * 64, col0 = (wg >> 1) * NW;
  const int q = et & 63, r0 = et >> 6;                  // this thread's output pixels: column q, rows r0 + 8*i, i = 0..7
  uint32_t si = 0, it = 0;   // si: running A-stage counter
  for (int w = blockIdx.x; w < total; w += gridDim.x, ++it) {
    const int n = w / 3, k = w % 3;
    float acc[8][2];
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc[i][0] = 0.f; acc[i][1] = 0.f; }
    mbar_wait(bfull_bar, it & 1u);
    for (int mt = 0; mt < kTilesPerImage; ++mt) {
      float am[NW / 2], ac[PASSES == 3 ? NW / 2 : 1];
#pragma unroll
      for (int j = 0; j < NW / 2; ++j) am[j] = 0.f;
#pragma unroll
      for (int j = 0; j < (PASSES == 3 ? NW / 2 : 1); ++j) ac[j] = 0.f;
      wgmma_fence_regs(am);
      if (PASSES == 3) wgmma_fence_regs(ac);
      for (int c = 0; c < 2; ++c, ++si) {
        const int s = si % kAStages;
        mbar_wait(full_bar(s), (si / kAStages) & 1u);
        const uint32_t sa = a_base + s * Cfg::kAStage + row0 * 128, sb = b_base + c * Cfg::kBChunk + col0 * 128;
        const uint64_t a_hi = make_sw128_desc(sa), a_lo = make_sw128_desc(sa + 128 * 64 * 2);
        const uint64_t b_hi = make_sw128_desc(sb), b_lo = make_sw128_desc(sb + BN * 64 * 2);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint64_t ko = (uint64_t)(kk * 2);
          const uint32_t a = (c > 0 || kk > 0) ? 1u : 0u;
          wgmma_bf16<NW>(am, a_hi + ko, b_hi + ko, a);
          if constexpr (PASSES == 3) {
            wgmma_bf16<NW>(ac, a_lo + ko, b_hi + ko, a);
            wgmma_bf16<NW>(ac, a_hi + ko, b_lo + ko, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(am);
        if (PASSES == 3) wgmma_fence_regs(ac);
        if (wtid == 0) mbar_arrive(empty_bar(s));       // this warpgroup no longer reads the stage
      }
      // T tile row = pixel (pr*64 + q) of input rows 2mt + pr; columns tap*2 + filter (66 used)
#pragma unroll
      for (int j = 0; j < NW / 2; ++j) {
        const int row = row0 + frag_row(wtid, j), col = col0 + frag_col(wtid, j);
        float v = am[j];
        if constexpr (PASSES == 3) v += ac[j];
        if (col < 2 * kNT) Ts[row * kTLd + col] = v;
      }
      asm volatile("bar.sync 1, 512;" ::: "memory");   // T tile complete (consumer warps only)
      if (mt == kTilesPerImage - 1 && threadIdx.x == 0) mbar_arrive(bempty_bar);   // every MMA of this item has retired

      // ha[p][f] += T[(p + dy, q + dx)][j*2 + f] for the taps whose input row p + dy lies in this tile (rows 2mt, 2mt+1).
      // The scales-[2,3,4] MDC has an analytic tap set (checked on the host against the sorted table): a row offset
      // dy != 0 belongs to exactly one dilation s = |dy| with dx in {-s, 0, +s} (T columns j0, j0+1, j0+2); dy = 0 has
      // dx in {-1,0,1,-2,2,-3,3,-4,4} (columns 12..20).  No table look-ups, independent loads per hit.
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int p = r0 + 8 * i;
#pragma unroll
        for (int pr = 0; pr < 2; ++pr) {
          const int dy = 2 * mt + pr - p;              // the row offset that reaches input row 2mt + pr from p (warp-uniform)
          if (dy < -4 || dy > 4) continue;
          const float* trow = Ts + (pr * 64 + q) * kTLd;
          if (dy != 0) {
            const int sdil = dy < 0 ? -dy : dy;
            const int j0 = dy < 0 ? 3 * (dy + 4) : 21 + 3 * (dy - 1);
            const float* tc0 = trow + 2 * j0;
            float a0 = tc0[2], a1 = tc0[3];            // dx = 0
            if (q - sdil >= 0) { a0 += tc0[-sdil * kTLd]; a1 += tc0[-sdil * kTLd + 1]; }          // dx = -s
            if (q + sdil <= 63) { a0 += tc0[sdil * kTLd + 4]; a1 += tc0[sdil * kTLd + 5]; }       // dx = +s
            acc[i][0] += a0;
            acc[i][1] += a1;
          } else {
            const float* tc0 = trow + 2 * 12;
            float a0 = tc0[2], a1 = tc0[3];            // dx = 0 (column 13)
#pragma unroll
            for (int e = 0; e < 4; ++e) {              // dx = -(e+1) / +(e+1): columns {12,14}, {15,16}, {17,18}, {19,20}
              const int d = e + 1;
              const int cm = e == 0 ? 0 : 2 * (2 * e + 1), cp = e == 0 ? 4 : 2 * (2 * e + 2);
              if (q - d >= 0) { a0 += tc0[-d * kTLd + cm]; a1 += tc0[-d * kTLd + cm + 1]; }
              if (q + d <= 63) { a0 += tc0[d * kTLd + cp]; a1 += tc0[d * kTLd + cp + 1]; }
            }
            acc[i][0] += a0;
            acc[i][1] += a1;
          }
        }
      }
      asm volatile("bar.sync 1, 512;" ::: "memory");   // T tile consumed: may be overwritten
    }
    float* o0 = ha + ((long long)n * 6 + 2 * k) * 4096 + q;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o0[(r0 + 8 * i) * 64] = acc[i][0];
      o0[4096 + (r0 + 8 * i) * 64] = acc[i][1];
    }
  }
}

}  // namespace

HeadMaps* head_build_maps(const __nv_bfloat16* fh4, long long fh4_plane, int n_img, const __nv_bfloat16* wt, long long wt_plane,
                          char* err, int errlen) {
  tc::EncodeTiledFn enc = tc::get_encode_fn();
  if (!enc) { snprintf(err, errlen, "cuTensorMapEncodeTiled entry point not available"); return nullptr; }
  HeadMaps* m = new HeadMaps();
  memset(m, 0, sizeof(*m));
  for (int planes = 2; planes >= 1; --planes) {
    {
      cuuint64_t dims[5] = {128, 64, 64, (cuuint64_t)n_img, 2};
      cuuint64_t strides[4] = {128 * 2, 64 * 128 * 2, 64 * 64 * 128 * 2, (cuuint64_t)fh4_plane * 2};
      cuuint32_t box[5] = {64, 64, 2, 1, (cuuint32_t)planes};
      cuuint32_t estr[5] = {1, 1, 1, 1, 1};
      CUresult r = enc(planes == 2 ? &m->a : &m->a1, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)fh4, dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(head A) failed: %d", (int)r); delete m; return nullptr; }
    }
    {
      cuuint64_t dims[3] = {128, 3 * BN, 2};
      cuuint64_t strides[2] = {128 * 2, (cuuint64_t)wt_plane * 2};
      cuuint32_t box[3] = {64, BN, (cuuint32_t)planes};
      cuuint32_t estr[3] = {1, 1, 1};
      CUresult r = enc(planes == 2 ? &m->b : &m->b1, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)wt, dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(head B) failed: %d", (int)r); delete m; return nullptr; }
    }
  }
  return m;
}

void head_free_maps(HeadMaps* m) { delete m; }

int launch_head_tc(const HeadMaps* maps, int passes, float* ha, int n, cudaStream_t st) {
  static DeviceOnce attr3, attr1;
  const int dev = cur_device();
  const int total = n * 3;
  const int num_sms = tc_num_sms();
  const int grid = total < num_sms ? total : num_sms;
  if (passes == 3) {
    if (!attr3.is_done(dev)) {
      if (cudaFuncSetAttribute(head_tc_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, HeadCfg<3>::kSmemBytes) != cudaSuccess) return -1;
      attr3.set_done(dev);
    }
    if (launch_pdl(head_tc_kernel<3>, dim3(grid), dim3(kThreads), HeadCfg<3>::kSmemBytes, st, *maps, ha, n) != cudaSuccess) return -1;
  } else {
    if (!attr1.is_done(dev)) {
      if (cudaFuncSetAttribute(head_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, HeadCfg<1>::kSmemBytes) != cudaSuccess) return -1;
      attr1.set_done(dev);
    }
    if (launch_pdl(head_tc_kernel<1>, dim3(grid), dim3(kThreads), HeadCfg<1>::kSmemBytes, st, *maps, ha, n) != cudaSuccess) return -1;
  }
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ian
