// wgrad_tc.cu -- weight gradient of a forward tap-GEMM (tapgemm.h: WgradGemm) on Hopper (sm_90a), its FFMA verification
// kernel and the ordered split-K finalize.
//
// The forward contracts over channels; its weight gradient contracts over PIXELS:
//   dB[t][co][ci] = sum_{n,p,q} G[n, p*osh+oh0, q*osw+ow0, co] * A[n, (p+dh_t)*sh+vh_t, (q+dw_t)*sw+vw_t, ci]
// Both operands arrive channel-contiguous, so with K = pixels they are MN-major for the MMA.  wgrad_tc_kernel:
//   warp 8     : TMA producer.  Per K step (64 pixels) four bulk-tensor loads of {64 ch, Wk, Hk, Nk, 2 planes} boxes:
//                G through the stride-osh parity view of the output gradient at the tap's phase offset (two boxes: the
//                tile's two 64-row halves of Cout), and A through the forward's shifted view (two boxes: the tile's 128
//                Cin columns) -- the conv padding is TMA's out-of-bounds fill, exactly as in the forward.  A box lands
//                as 64 pixel rows of 64 channels with the 128B swizzle: an MN-major wgmma operand, no transpose pass.
//   warps 0..7 : two consumer warpgroups, one per 64-row half of the Cout tile; wgmma with the transpose immediates,
//                float32 fidelity from bf16 hi|lo planes as in tapgemm_tc.cu (main += G_hi*A_hi,
//                cross += G_lo*A_hi + G_hi*A_lo, one add at the end), then the raw sums go to this K split's slab.
// Persistent CTAs walk (tap | m-tile | n-tile | k-split) work items; the 3-stage operand ring runs across items.
#include <cuda.h>

#include <cstdio>
#include <cstring>

#include "tapgemm.h"
#include "tc_ptx.cuh"

namespace ian {

struct WgradMaps {
  CUtensorMap g[kMaxPhases];   // output-gradient parity views, box = {64 ch, Wk, Hk, Nk, 2 planes}
  CUtensorMap a[4];            // activation views (the forward's), same box
  int Wk, Hk, Nk, kboxes;      // a K step is a {Nk images, Hk rows, Wk cols} box of the phase grid
  int ntaps;
};

namespace {

using namespace tc;

constexpr int WBM = 128, WBN = 128, WBK = 64;   // Cout rows, Cin columns, pixels per K step
constexpr int kBoxBytes = 64 * WBK * 2 * 2;      // {64 ch, 64 px, hi|lo}: 16 KB
constexpr int kStageBytes = 4 * kBoxBytes;       // two G boxes + two A boxes
constexpr int kStages = 3;
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int kThreadsCta = 288;

// pixel boxes of WBK pixels tiling the (n, p, q) grid
void k_box_shape(int Hg, int Wg, int& Wk, int& Hk, int& Nk) {
  Wk = Wg < WBK ? Wg : WBK;
  Hk = Hg < WBK / Wk ? Hg : WBK / Wk;
  Nk = WBK / (Wk * Hk);
}

struct WItem { int ti, ph, mt, nt, ks, j0, j1; };

__device__ __forceinline__ WItem wgrad_item(const WgradGemm& w, const WgradMaps& m, int idx) {
  WItem it;
  const int tiles_m = w.f.Cout / WBM, tiles_n = w.f.Cin / WBN;
  it.ti = idx % m.ntaps; idx /= m.ntaps;
  it.mt = idx % tiles_m; idx /= tiles_m;
  it.nt = idx % tiles_n; idx /= tiles_n;
  it.ks = idx;
  it.ph = 0;
  while (it.ph + 1 < w.f.nphase && it.ti >= w.f.phase[it.ph + 1].tap_begin) ++it.ph;
  it.j0 = (int)((long long)m.kboxes * it.ks / w.ksplit);
  it.j1 = (int)((long long)m.kboxes * (it.ks + 1) / w.ksplit);
  return it;
}

__global__ void __launch_bounds__(kThreadsCta, 1)
wgrad_tc_kernel(const __grid_constant__ WgradGemm w, const __grid_constant__ WgradMaps m, const int total_work) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + kStages * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  const int warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    pdl_trigger();
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);                       // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                                           // every operand is an activation of this chain (tapgemm.h: PDL)
  const int qboxes = w.f.Wg / m.Wk, pboxes = w.f.Hg / m.Hk;

  if (warp == 8) {
    // ===================== TMA producer =====================
    uint32_t i = 0;
    for (int wi = blockIdx.x; wi < total_work; wi += gridDim.x) {
      const WItem it = wgrad_item(w, m, wi);
      const Tap tap = w.f.taps[it.ti];
      for (int j = it.j0; j < it.j1; ++j, ++i) {
        const int s = i % kStages;
        const uint32_t par = (i / kStages) & 1u;
        const int q0 = (j % qboxes) * m.Wk, p0 = ((j / qboxes) % pboxes) * m.Hk, n0 = j / (qboxes * pboxes) * m.Nk;
        mbar_wait(empty_bar(s), par ^ 1u);
        const uint32_t sa = smem_base + s * kStageBytes;
        if (elect_one_sync()) {
          mbar_expect_tx(full_bar(s), kStageBytes);
          tma_load_5d(&m.g[it.ph], full_bar(s), sa, it.mt * WBM, q0, p0, n0, 0);
          tma_load_5d(&m.g[it.ph], full_bar(s), sa + kBoxBytes, it.mt * WBM + 64, q0, p0, n0, 0);
          tma_load_5d(&m.a[tap.view], full_bar(s), sa + 2 * kBoxBytes, it.nt * WBN, q0 + tap.dw, p0 + tap.dh, n0, 0);
          tma_load_5d(&m.a[tap.view], full_bar(s), sa + 3 * kBoxBytes, it.nt * WBN + 64, q0 + tap.dw, p0 + tap.dh, n0, 0);
        }
        __syncwarp();
      }
    }
    return;
  }

  // ===================== consumers: 64 Cout rows x 128 Cin columns per warpgroup =====================
  const int wg = warp >> 2, wtid = threadIdx.x & 127;
  uint32_t i = 0;
  for (int wi = blockIdx.x; wi < total_work; wi += gridDim.x) {
    const WItem it = wgrad_item(w, m, wi);
    float acc_m[64], acc_c[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) { acc_m[j] = 0.f; acc_c[j] = 0.f; }
    wgmma_fence_regs(acc_m);
    wgmma_fence_regs(acc_c);
    for (int j = it.j0; j < it.j1; ++j, ++i) {
      const int s = i % kStages;
      mbar_wait(full_bar(s), (i / kStages) & 1u);
      const uint32_t sa = smem_base + s * kStageBytes;
      const uint32_t ga = sa + wg * kBoxBytes, aa = sa + 2 * kBoxBytes;
      const uint64_t g_hi = make_sw128_mn_desc(ga, 0), g_lo = make_sw128_mn_desc(ga + kBoxBytes / 2, 0);
      const uint64_t a_hi = make_sw128_mn_desc(aa, kBoxBytes), a_lo = make_sw128_mn_desc(aa + kBoxBytes / 2, kBoxBytes);
      const uint32_t first = (j == it.j0) ? 0u : 1u;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < WBK / 16; ++k) {
        const uint64_t ko = (uint64_t)(k * 128);       // 16 pixel rows = two 1024-byte K groups, in 16-byte units
        const uint32_t acc = k > 0 ? 1u : first;
        wgmma_bf16_mn<128>(acc_m, g_hi + ko, a_hi + ko, acc);
        wgmma_bf16_mn<128>(acc_c, g_lo + ko, a_hi + ko, acc);
        wgmma_bf16_mn<128>(acc_c, g_hi + ko, a_lo + ko, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();                                  // the previous K step's MMAs have retired: free its stage
      if (j > it.j0 && wtid == 0) mbar_arrive(empty_bar((i - 1) % kStages));
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc_m);
    wgmma_fence_regs(acc_c);
    if (it.j1 > it.j0 && wtid == 0) mbar_arrive(empty_bar((i - 1) % kStages));
#pragma unroll
    for (int j = 0; j < 64; ++j) acc_m[j] += acc_c[j];
    const Tap tap = w.f.taps[it.ti];
    float* slab = w.ws + (long long)it.ks * w.ws_slab +
                  ((long long)tap.wtile * w.f.Cout + it.mt * WBM + wg * 64) * w.f.Cin + it.nt * WBN;
#pragma unroll
    for (int j = 0; j < 64; j += 2)
      __stcg(reinterpret_cast<float2*>(slab + (long long)frag_row(wtid, j) * w.f.Cin + frag_col(wtid, j)),
             make_float2(acc_m[j], acc_m[j + 1]));
  }
}

// ---- verification path: FFMA on the re-joined float32 operands, 64 x 64 output tiles, 16 pixels per step ----
__device__ __forceinline__ float4 join4(const __nv_bfloat16* hi, long long plane) {
  const uint2 h = *reinterpret_cast<const uint2*>(hi);
  const uint2 l = *reinterpret_cast<const uint2*>(hi + plane);
  const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&h);
  const __nv_bfloat162* lp = reinterpret_cast<const __nv_bfloat162*>(&l);
  const float2 h0 = __bfloat1622float2(hp[0]), h1 = __bfloat1622float2(hp[1]);
  const float2 l0 = __bfloat1622float2(lp[0]), l1 = __bfloat1622float2(lp[1]);
  return make_float4(h0.x + l0.x, h0.y + l0.y, h1.x + l1.x, h1.y + l1.y);
}

__global__ void __launch_bounds__(256) wgrad_simt_kernel(const __grid_constant__ WgradGemm w, int ntaps) {
  __shared__ __align__(16) float Gs[16][64 + 4];
  __shared__ __align__(16) float As[16][64 + 4];
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const TapGemm& f = w.f;
  const int ci0 = blockIdx.x * 64, co0 = blockIdx.y * 64;
  const int ti = blockIdx.z % ntaps, ks = blockIdx.z / ntaps;
  int ph = 0;
  while (ph + 1 < f.nphase && ti >= f.phase[ph + 1].tap_begin) ++ph;
  const Tap tap = f.taps[ti];
  const int oh0 = f.phase[ph].oh0, ow0 = f.phase[ph].ow0;
  const long long M = (long long)f.n_img * f.Hg * f.Wg;
  const long long m0 = M * ks / w.ksplit, m1 = M * (ks + 1) / w.ksplit;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int lr = tid >> 4, lc = (tid & 15) * 4;
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  for (long long mb = m0; mb < m1; mb += 16) {
    const long long mm = mb + lr;
    float4 gv = make_float4(0.f, 0.f, 0.f, 0.f), av = gv;
    if (mm < m1) {
      const int q = (int)(mm % f.Wg), p = (int)((mm / f.Wg) % f.Hg), n = (int)(mm / ((long long)f.Wg * f.Hg));
      const long long gpix = ((long long)n * f.Hout + p * f.osh + oh0) * f.Wout + q * f.osw + ow0;
      gv = join4(w.gr + gpix * f.Cout + co0 + lc, w.gr_plane);
      const int vp = p + tap.dh, vq = q + tap.dw;
      const int ih = vp * f.sh + (tap.view >> 1), iw = vq * f.sw + (tap.view & 1);
      if (vp >= 0 && vq >= 0 && ih < f.Hin && iw < f.Win)
        av = join4(f.a + ((long long)(n * f.Hin + ih) * f.Win + iw) * f.Cin + ci0 + lc, f.a_plane);
    }
    __syncthreads();
    *reinterpret_cast<float4*>(&Gs[lr][lc]) = gv;
    *reinterpret_cast<float4*>(&As[lr][lc]) = av;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float4 g4 = *reinterpret_cast<const float4*>(&Gs[kk][ty * 4]);
      const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][tx * 4]);
      const float gr[4] = {g4.x, g4.y, g4.z, g4.w}, ar[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(gr[a], ar[b], acc[a][b]);
    }
  }
  float* slab = w.ws + (long long)ks * w.ws_slab + ((long long)tap.wtile * f.Cout + co0 + ty * 4) * f.Cin + ci0 + tx * 4;
#pragma unroll
  for (int a = 0; a < 4; ++a)
    *reinterpret_cast<float4*>(slab + (long long)a * f.Cin) = make_float4(acc[a][0], acc[a][1], acc[a][2], acc[a][3]);
}

// slabs [ksplit][ntiles][Cout][Cin] -> sum in split order -> reference layout (out = sum, or out += sum for a later batch
// chunk).  One thread per slab element: the slab reads are coalesced, the scattered write happens once.
__global__ void __launch_bounds__(256) wgrad_finalize_kernel(const float* __restrict__ ws, int ksplit, long long slab,
                                                             int layout, int Cout, int Cin, float* __restrict__ out,
                                                             int accumulate) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= slab) return;
  const int ci = (int)(idx % Cin);
  const int co = (int)((idx / Cin) % Cout);
  const int t = (int)(idx / ((long long)Cin * Cout));
  long long dst;
  if (layout == WG_FC2) {
    if (ci >= 100) return;                              // z padded 100 -> 128
    const int hw = co / 1024, c = co % 1024;
    dst = (long long)ci * 16384 + c * 16 + hw;
  } else {
    dst = ((long long)ci * Cout + co) * 25 + t;
  }
  float a = __ldcg(ws + idx);
  for (int k = 1; k < ksplit; ++k) a += __ldcg(ws + (long long)k * slab + idx);
  out[dst] = accumulate ? out[dst] + a : a;
}

}  // namespace

WgradMaps* wgrad_build_maps(const WgradGemm& w, char* err, int errlen) {
  const TapGemm& f = w.f;
  tc::EncodeTiledFn enc = tc::get_encode_fn();
  if (!enc) { snprintf(err, errlen, "cuTensorMapEncodeTiled entry point not available"); return nullptr; }
  if (f.Cin % WBN || f.Cout % WBM) { snprintf(err, errlen, "wgrad needs Cin %% 128 == 0 and Cout %% 128 == 0 (got %d, %d)", f.Cin, f.Cout); return nullptr; }
  WgradMaps* m = new WgradMaps();
  memset(m, 0, sizeof(*m));
  k_box_shape(f.Hg, f.Wg, m->Wk, m->Hk, m->Nk);
  if (f.Wg % m->Wk || f.Hg % m->Hk || m->Wk * m->Hk * m->Nk != WBK) {
    snprintf(err, errlen, "M grid %dx%d does not tile into 64-pixel boxes", f.Hg, f.Wg);
    delete m; return nullptr;
  }
  m->kboxes = (f.Wg / m->Wk) * (f.Hg / m->Hk) * ((f.n_img + m->Nk - 1) / m->Nk);
  m->ntaps = f.phase[f.nphase - 1].tap_begin + f.phase[f.nphase - 1].ntaps;
  // each weight tile in exactly one (phase, tap): the per-tap GEMMs then write disjoint slab tiles
  {
    int seen[kMaxTaps] = {0};
    for (int t = 0; t < m->ntaps; ++t) {
      const int wt = f.taps[t].wtile;
      if (wt < 0 || wt >= kMaxTaps || seen[wt]++) {
        snprintf(err, errlen, "weight tile %d is used by more than one tap", wt);
        delete m; return nullptr;
      }
    }
  }
  cuuint32_t box[5] = {64, (cuuint32_t)m->Wk, (cuuint32_t)m->Hk, (cuuint32_t)m->Nk, 2};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  for (int p = 0; p < f.nphase; ++p) {
    cuuint64_t dims[5] = {(cuuint64_t)f.Cout, (cuuint64_t)f.Wg, (cuuint64_t)f.Hg, (cuuint64_t)f.n_img, 2};
    cuuint64_t strides[4] = {(cuuint64_t)f.osw * f.Cout * 2, (cuuint64_t)f.osh * f.Wout * f.Cout * 2,
                             (cuuint64_t)f.Hout * f.Wout * f.Cout * 2, (cuuint64_t)w.gr_plane * 2};
    void* base = (void*)(w.gr + ((long long)f.phase[p].oh0 * f.Wout + f.phase[p].ow0) * f.Cout);
    CUresult r = enc(&m->g[p], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(G phase %d) failed: %d", p, (int)r); delete m; return nullptr; }
  }
  bool used[4] = {false, false, false, false};
  for (int t = 0; t < m->ntaps; ++t) used[f.taps[t].view] = true;
  for (int v = 0; v < 4; ++v) {
    if (!used[v]) continue;
    const int vh = v >> 1, vw = v & 1;
    const cuuint64_t Hv = (f.Hin - vh + f.sh - 1) / f.sh, Wv = (f.Win - vw + f.sw - 1) / f.sw;
    cuuint64_t dims[5] = {(cuuint64_t)f.Cin, Wv, Hv, (cuuint64_t)f.n_img, 2};
    cuuint64_t strides[4] = {(cuuint64_t)f.sw * f.Cin * 2, (cuuint64_t)f.sh * f.Win * f.Cin * 2,
                             (cuuint64_t)f.Hin * f.Win * f.Cin * 2, (cuuint64_t)f.a_plane * 2};
    void* base = (void*)(f.a + ((long long)vh * f.Win + vw) * f.Cin);
    CUresult r = enc(&m->a[v], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(A view %d) failed: %d", v, (int)r); delete m; return nullptr; }
  }
  return m;
}

void wgrad_free_maps(WgradMaps* m) { delete m; }

int wgrad_kboxes(const WgradGemm& w) {
  int Wk, Hk, Nk;
  k_box_shape(w.f.Hg, w.f.Wg, Wk, Hk, Nk);
  return (w.f.Wg / Wk) * (w.f.Hg / Hk) * ((w.f.n_img + Nk - 1) / Nk);
}

// Split K (pixels) when the layer has few output tiles (dec_conv3: 25 taps x 1 x 2 tiles, K = n*256 per tap): pick the
// split count in 1..16 with the shortest makespan in tile units, ceil(items / SMs) / ksplit, keeping >= 2 K steps per
// split and ksplit * slab <= max_ws_floats.  Depends only on the plan's batch and the SM count.
int wgrad_choose_ksplit(const WgradGemm& w, long long max_ws_floats) {
  const int sms = tc_num_sms();
  const int kb = wgrad_kboxes(w);
  const long long tiles = (long long)(w.f.Cout / WBM) * (w.f.Cin / WBN) * (w.f.phase[w.f.nphase - 1].tap_begin + w.f.phase[w.f.nphase - 1].ntaps);
  int best = 1;
  double best_cost = (double)((tiles + sms - 1) / sms);
  for (int ks = 2; ks <= 16 && 2 * ks <= kb; ++ks) {
    if ((long long)ks * w.ws_slab > max_ws_floats) break;
    const double cost = (double)((tiles * ks + sms - 1) / sms) / ks;
    if (cost < best_cost * 0.98) { best = ks; best_cost = cost; }
  }
  return best;
}

int launch_wgrad_tc(const WgradGemm& w, const WgradMaps* maps, cudaStream_t st) {
  static DeviceOnce attr_set;
  const int dev = cur_device();
  if (!attr_set.is_done(dev)) {
    if (cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess) return -1;
    attr_set.set_done(dev);
  }
  const int total = maps->ntaps * (w.f.Cout / WBM) * (w.f.Cin / WBN) * w.ksplit;
  const int grid = total < tc_num_sms() ? total : tc_num_sms();
  if (launch_pdl(wgrad_tc_kernel, dim3(grid), dim3(kThreadsCta), kSmemBytes, st, w, *maps, total) != cudaSuccess) return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_wgrad_simt(const WgradGemm& w, cudaStream_t st) {
  const int ntaps = w.f.phase[w.f.nphase - 1].tap_begin + w.f.phase[w.f.nphase - 1].ntaps;
  if (launch_pdl(wgrad_simt_kernel, dim3(w.f.Cin / 64, w.f.Cout / 64, ntaps * w.ksplit), dim3(256), 0, st, w, ntaps) != cudaSuccess)
    return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_wgrad_finalize(const WgradGemm& w, int layout, float* out, int accumulate, cudaStream_t st) {
  if (launch_pdl(wgrad_finalize_kernel, dim3((unsigned)((w.ws_slab + 255) / 256)), dim3(256), 0, st, (const float*)w.ws,
                 w.ksplit, w.ws_slab, layout, w.f.Cout, w.f.Cin, out, accumulate) != cudaSuccess)
    return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ian
