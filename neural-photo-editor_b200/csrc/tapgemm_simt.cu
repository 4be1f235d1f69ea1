// tapgemm_simt.cu -- fp32 FFMA implementation of the shifted-tap GEMM (see tapgemm.h).
// This is the verification path (IAN_PATH_SIMT): it shares no arithmetic with the wgmma kernel
// (operands are re-joined to fp32, products and sums are plain FFMA), so the two check each other on
// the GPU.  Also hosts the split-K finalize kernel used by the tensor-core path.
#include "tapgemm.h"

namespace ian {

namespace {

constexpr int BM = 64, BN = 64, BK = 16;   // Cout may be 16 (RGB-Beta head): columns >= Cout are masked

__device__ __forceinline__ float4 load_join4(const __nv_bfloat16* hi, long long plane, bool use_lo) {
  // 4 consecutive channels: hi and lo planes, 8 bytes each (lo ignored in single-pass bf16 mode)
  uint2 h = *reinterpret_cast<const uint2*>(hi);
  uint2 l = use_lo ? *reinterpret_cast<const uint2*>(hi + plane) : make_uint2(0u, 0u);
  const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&h);
  const __nv_bfloat162* lp = reinterpret_cast<const __nv_bfloat162*>(&l);
  float2 h0 = __bfloat1622float2(hp[0]), h1 = __bfloat1622float2(hp[1]);
  float2 l0 = __bfloat1622float2(lp[0]), l1 = __bfloat1622float2(lp[1]);
  return make_float4(h0.x + l0.x, h0.y + l0.y, h1.x + l1.x, h1.y + l1.y);
}

__device__ __forceinline__ void epilogue_store(const TapGemm& g, float acc, long long pix, int oh, int ow,
                                               int co, __nv_bfloat16* hi4, __nv_bfloat16* lo4,
                                               float* f4, int j) {
  int si = co + (oh * g.Wout + ow) * g.scale_pix_stride;
  float sc = g.scale ? g.scale[si] : 1.f;
  float v;
  if (g.out_raw) {
    __nv_bfloat16 rh, rl;
    split_bf16(acc, rh, rl);
    g.out_raw[pix * g.Cout + co] = rh;
    if (g.passes != 1) g.out_raw[g.out_raw_plane + pix * g.Cout + co] = rl;
  }
  const float resv = g.res ? __bfloat162float(g.res[pix * g.Cout + co]) + (g.passes != 1 ? __bfloat162float(g.res[g.res_plane + pix * g.Cout + co]) : 0.f) : 0.f;
  if (!g.res_after) acc += resv;
  if (g.act == ACT_MASK) {
    float mk = __bfloat162float(g.mask[pix * g.Cout + co]);
    v = mk > 0.f ? acc * sc : acc * sc * g.mask_slope;
    if (g.res_after) v += resv;
  } else {
    float sf = g.shift ? g.shift[si] : 0.f;
    v = act_apply(fmaf(acc, sc, sf), g.act);
  }
  f4[j] = v;
  split_bf16(v, hi4[j], lo4[j]);
}

__global__ void __launch_bounds__(256) tapgemm_simt_kernel(const __grid_constant__ TapGemm g) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const Phase ph = g.phase[blockIdx.z];
  const int M = g.n_img * g.Hg * g.Wg;

  // the row this thread loads for A
  const int lr = tid >> 2, lc = (tid & 3) * 4;
  const int lm = m0 + lr;
  int ln = 0, lp = 0, lq = 0;
  const bool lvalid = lm < M;
  if (lvalid) {
    lq = lm % g.Wg;
    int t = lm / g.Wg;
    lp = t % g.Hg;
    ln = t / g.Hg;
  }

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int t = 0; t < ph.ntaps; ++t) {
    const Tap tap = g.taps[ph.tap_begin + t];
    const int vp = lp + tap.dh, vq = lq + tap.dw;
    const int ih = vp * g.sh + (tap.view >> 1), iw = vq * g.sw + (tap.view & 1);
    const bool ok = lvalid && vp >= 0 && vq >= 0 && ih < g.Hin && iw < g.Win;
    const __nv_bfloat16* arow =
        g.a + ((long long)(ln * g.Hin + ih) * g.Win + iw) * g.Cin + lc;
    const __nv_bfloat16* brow =
        g.b + ((long long)tap.wtile * g.Cout + (n0 + lr)) * g.Cin + lc;
    for (int c0 = 0; c0 < g.Cin; c0 += BK) {
      float4 av = ok ? load_join4(arow + c0, g.a_plane, g.passes != 1) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 bv = (n0 + lr < g.Cout) ? load_join4(brow + c0, g.b_plane, g.passes != 1) : make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
      As[lc + 0][lr] = av.x; As[lc + 1][lr] = av.y; As[lc + 2][lr] = av.z; As[lc + 3][lr] = av.w;
      Bs[lc + 0][lr] = bv.x; Bs[lc + 1][lr] = bv.y; Bs[lc + 2][lr] = bv.z; Bs[lc + 3][lr] = bv.w;
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        float ar[4] = {a4.x, a4.y, a4.z, a4.w};
        float br[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
      }
    }
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const int q = m % g.Wg;
    const int t2 = m / g.Wg;
    const int p = t2 % g.Hg, n = t2 / g.Hg;
    const int oh = p * g.osh + ph.oh0, ow = q * g.osw + ph.ow0;
    const long long pix = (long long)(n * g.Hout + oh) * g.Wout + ow;
    const int co = n0 + tx * 4;
    if (co >= g.Cout) continue;
    __align__(8) __nv_bfloat16 hi4[4], lo4[4];
    __align__(16) float f4[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) epilogue_store(g, acc[i][j], pix, oh, ow, co + j, hi4, lo4, f4, j);
    if (g.out) {
      *reinterpret_cast<uint2*>(g.out + pix * g.Cout + co) = *reinterpret_cast<uint2*>(hi4);
      if (g.passes != 1) *reinterpret_cast<uint2*>(g.out + g.out_plane + pix * g.Cout + co) = *reinterpret_cast<uint2*>(lo4);
    }
    if (g.out_f32) *reinterpret_cast<float4*>(g.out_f32 + pix * g.Cout + co) = *reinterpret_cast<float4*>(f4);
    if (g.out_f32_t) {                                     // same tile-blocked layout as the tensor-core kernel
      int Wt, Ht, Nt;
      tile_shape(g.Hg, g.Wg, Wt, Ht, Nt);
      const int tq = g.Wg / Wt, tp = g.Hg / Ht;
      const long long mtile = ((long long)(n / Nt) * tp + p / Ht) * tq + q / Wt;
      const int ml = ((n % Nt) * Ht + p % Ht) * Wt + q % Wt;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (co + j < g.cout_real) {
          const long long ti = (mtile * g.cout_real + co + j) * 128 + ml;
          if (g.out_t_bf16) reinterpret_cast<__nv_bfloat16*>(g.out_f32_t)[ti] = __float2bfloat16_rn(f4[j]);
          else g.out_f32_t[ti] = f4[j];
        }
    }
  }
}

// ws[split][pix][Cout] raw accumulators -> sum over splits -> epilogue -> planes / f32.  One thread per 4 channels.
__global__ void __launch_bounds__(256) splitk_finalize_kernel(const __grid_constant__ TapGemm g, long long npix) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c4 = g.Cout / 4;
  if (idx >= npix * c4) return;
  const long long pix = idx / c4;
  const int co = (int)(idx % c4) * 4;
  const int ow = (int)(pix % g.Wout);
  const int oh = (int)((pix / g.Wout) % g.Hout);
  const float* wp = g.ws + pix * g.Cout + co;
  float4 a = __ldcg(reinterpret_cast<const float4*>(wp));
  int k = 1;
  for (; k + 8 <= g.ksplit; k += 8) {                      // 8 slab loads in flight, added in split order: bit-reproducible
    float4 b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] = __ldcg(reinterpret_cast<const float4*>(wp + (long long)(k + j) * g.ws_slab));
#pragma unroll
    for (int j = 0; j < 8; ++j) { a.x += b[j].x; a.y += b[j].y; a.z += b[j].z; a.w += b[j].w; }
  }
  for (; k < g.ksplit; ++k) {
    const float4 b = __ldcg(reinterpret_cast<const float4*>(wp + (long long)k * g.ws_slab));
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
  }
  float ar[4] = {a.x, a.y, a.z, a.w};
  __align__(8) __nv_bfloat16 hi4[4], lo4[4];
  __align__(16) float f4[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) epilogue_store(g, ar[j], pix, oh, ow, co + j, hi4, lo4, f4, j);
  if (g.out) {
    *reinterpret_cast<uint2*>(g.out + pix * g.Cout + co) = *reinterpret_cast<uint2*>(hi4);
    *reinterpret_cast<uint2*>(g.out + g.out_plane + pix * g.Cout + co) = *reinterpret_cast<uint2*>(lo4);
  }
  if (g.out_f32) *reinterpret_cast<float4*>(g.out_f32 + pix * g.Cout + co) = *reinterpret_cast<float4*>(f4);
}


// The same for deep splits (ksplit >= 8: the dense layers whose K = 16384 is spread over 18-64 CTAs).  One thread walking
// 64 slabs is a chain of L2 round trips on 16 thread blocks (18 us for the 128 x 128 output of the brush's dz GEMM); here
// 8 neighbouring lanes LOAD every 8th slab each (all loads in flight at once) and the values are then added in slab
// order 0, 1, 2, ... through shuffles -- the same float32 additions in the same order as the one-thread form, so the
// result is bit-identical to it (a shuffle tree would be a different rounding, and 16-bit activations downstream turn
// last-bit differences into ReLU-mask flips: DESIGN.md section 3).
__global__ void __launch_bounds__(256) splitk_finalize8_kernel(const __grid_constant__ TapGemm g, long long npix) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const long long gidx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int sub = threadIdx.x & 7;
  const int c4 = g.Cout / 4;
  const long long total = npix * c4;
  long long idx = gidx >> 3;
  const bool valid = idx < total;
  if (!valid) idx = total - 1;                          // keep the whole warp in the shuffles
  const long long pix = idx / c4;
  const int co = (int)(idx % c4) * 4;
  const float* wp = g.ws + pix * g.Cout + co;
  float4 b[8];                                          // slab r*8 + sub (ksplit <= 64)
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int k = r * 8 + sub;
    b[r] = k < g.ksplit ? __ldcg(reinterpret_cast<const float4*>(wp + (long long)k * g.ws_slab)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float4 a;                                             // starts as slab 0
  a.x = __shfl_sync(0xffffffffu, b[0].x, 0, 8);
  a.y = __shfl_sync(0xffffffffu, b[0].y, 0, 8);
  a.z = __shfl_sync(0xffffffffu, b[0].z, 0, 8);
  a.w = __shfl_sync(0xffffffffu, b[0].w, 0, 8);
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    if (r * 8 >= g.ksplit) break;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (r == 0 && j == 0) continue;
      if (r * 8 + j >= g.ksplit) break;                   // (warp-uniform)
      a.x += __shfl_sync(0xffffffffu, b[r].x, j, 8);
      a.y += __shfl_sync(0xffffffffu, b[r].y, j, 8);
      a.z += __shfl_sync(0xffffffffu, b[r].z, j, 8);
      a.w += __shfl_sync(0xffffffffu, b[r].w, j, 8);
    }
  }
  if (sub != 0 || !valid) return;
  const int ow = (int)(pix % g.Wout);
  const int oh = (int)((pix / g.Wout) % g.Hout);
  float ar[4] = {a.x, a.y, a.z, a.w};
  __align__(8) __nv_bfloat16 hi4[4], lo4[4];
  __align__(16) float f4[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) epilogue_store(g, ar[j], pix, oh, ow, co + j, hi4, lo4, f4, j);
  if (g.out) {
    *reinterpret_cast<uint2*>(g.out + pix * g.Cout + co) = *reinterpret_cast<uint2*>(hi4);
    *reinterpret_cast<uint2*>(g.out + g.out_plane + pix * g.Cout + co) = *reinterpret_cast<uint2*>(lo4);
  }
  if (g.out_f32) *reinterpret_cast<float4*>(g.out_f32 + pix * g.Cout + co) = *reinterpret_cast<float4*>(f4);
}

}  // namespace

int launch_tapgemm_simt(const TapGemm& g, cudaStream_t st) {
  const int M = g.n_img * g.Hg * g.Wg;
  dim3 grid((M + BM - 1) / BM, (g.Cout + BN - 1) / BN, g.nphase);
  tapgemm_simt_kernel<<<grid, 256, 0, st>>>(g);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_splitk_finalize(const TapGemm& g, cudaStream_t st) {
  const long long npix = (long long)g.n_img * g.Hout * g.Wout;
  const long long total = npix * (g.Cout / 4);
  if (coop_finalize_flag() && g.ksplit >= 8 && total <= 16384) {                 // few outputs, many slabs (the one-thread form fills <= 64 thread blocks)
    if (launch_pdl(splitk_finalize8_kernel, dim3((unsigned)((total * 8 + 255) / 256)), dim3(256), 0, st, g, npix) != cudaSuccess) return -1;
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
  }
  if (launch_pdl(splitk_finalize_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, g, npix) != cudaSuccess) return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ian
