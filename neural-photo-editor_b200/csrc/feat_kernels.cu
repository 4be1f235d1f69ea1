// feat_kernels.cu -- the IAN's introspection features and the latent fit under its feature-wise loss
// (ian_introspect_*, ian_introspect_jvp_*, ian_feature_gauss_newton_*, ian_fit_latent_features_*; DESIGN section 5.6k).
// The features g_1..g_4 are the encoder's stored activation planes a1..a4 (after BatchNorm and LeakyReLU), M_i = 131072,
// 65536, 32768, 16384 elements per image.  A feature value is what the encoder stores: hi + lo of the split planes (float32
// mode, exact in float32) or hi alone (bf16 mode).
//   feat_store        : split planes NHWC -> float32, NHWC (the fit's stored features) or NCHW (the reference layout)
//   feat_gram         : per sample, partial sums over 1024-element chunks of the upper triangle of [J_i | r_i]^T [J_i | r_i],
//                       J_i the 100 tangent rows of layer i (the batch-100 plan's tangent planes), r_i = g_i(x_hat) - g_i(x);
//                       float64 DFMA, register-tiled: every thread owns one 8 x 8 tile of the 104 x 104 (101 used) Gram
//   feat_gram_reduce  : A = sum_i c_i (chunk sums of layer i, in chunk order) [+ a A_pixel], likewise g and e
//   feat_accept       : e_trial = a |x_hat_trial - x|^2 + sum_i c_i |g_i(x_hat_trial) - g_i(x)|^2 in a fixed order, then
//                       gn_accept's rule; an accepted step (and the start) also keeps the trial's features as the current ones
//   feat_cotangent    : the features' cotangents (ian_introspect_vjp_*) float32 NCHW -> split planes NHWC, transposed
//                       through shared memory; the deepest supplied layer gets the backward GEMMs' ACT_MASK rule
// Every product of two operands is formed in float64, where a product of two float32 values is exact; the only roundings
// are the additions (in a fixed order) and the c_i and a scalings, applied once per layer sum.
#include "edge.h"

namespace ian {

namespace {

constexpr int kPix = 12288;
constexpr int kLat = 100;
constexpr int kRows = 104;              // 100 tangent rows, the residual row, 3 zero rows
constexpr int kTile = 8;                // each thread: one 8 x 8 tile of the Gram
constexpr int kTB = kRows / kTile;      // 13 tile rows
constexpr int kTiles = kTB * (kTB + 1) / 2;   // 91 tiles of the upper triangle
constexpr int kGramThreads = 96;
constexpr int kChunk = 1024;            // feature elements per CTA
constexpr int kSlab = 32;               // feature elements staged in shared memory per step
constexpr int kChunks = kFeatTotal / kChunk;   // 240: 128, 64, 32 and 16 per layer

__host__ __device__ __forceinline__ int chunk0(int l) { return 256 - (256 >> l); }   // first chunk of layer l (l = 4: the end)
__device__ __forceinline__ int layer_of_chunk(int c) { return c < 128 ? 0 : c < 192 ? 1 : c < 224 ? 2 : 3; }

// element l of a kernel-parameter array without a local copy of the array
template <typename T>
__device__ __forceinline__ T pick(const T (&v)[4], int l) { return l == 0 ? v[0] : l == 1 ? v[1] : l == 2 ? v[2] : v[3]; }

__device__ __forceinline__ float plane_value(const __nv_bfloat16* p, long long plane, int passes, long long i) {
  const float hi = __bfloat162float(p[i]);
  return passes == 1 ? hi : hi + __bfloat162float(p[plane + i]);
}

__global__ void __launch_bounds__(256) feat_store_kernel(const __nv_bfloat16* __restrict__ p, long long plane, int passes, int C,
                                                         int HW, long long total, float* __restrict__ out, int nchw) {
  pdl_trigger();
  pdl_wait();
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total; o += (long long)gridDim.x * blockDim.x) {
    long long i = o;
    if (nchw) {                                           // o = (k * C + c) * HW + s  <-  i = (k * HW + s) * C + c
      const long long s = o % HW, c = (o / HW) % C, k = o / ((long long)HW * C);
      i = (k * HW + s) * C + c;
    }
    out[o] = plane_value(p, plane, passes, i);
  }
}

// grid kChunks, kGramThreads; part[chunk][tile][8][8]
__global__ void __launch_bounds__(kGramThreads, 2) feat_gram_kernel(FeatLayers t, int passes, double* __restrict__ part) {
  pdl_trigger();
  __shared__ __align__(16) double s[kSlab][kRows];
  const int chunk = blockIdx.x, tid = threadIdx.x;
  const int l = layer_of_chunk(chunk);
  const long long M = feat_m(l);
  const long long k0 = (long long)(chunk - chunk0(l)) * kChunk;
  const __nv_bfloat16* tp = pick(t.tan, l);
  const long long plane = pick(t.plane, l);
  const float* cur = pick(t.cur, l);
  const float* tgt = pick(t.tgt, l);
  int ti = 0, q = tid;
  while (ti < kTB && q >= kTB - ti) { q -= kTB - ti; ++ti; }
  const bool live = tid < kTiles;
  const int tj = ti + q;
  for (int e = tid; e < kSlab * (kRows - kLat - 1); e += kGramThreads)   // the zero rows 101..103, never overwritten
    s[e % kSlab][kLat + 1 + e / kSlab] = 0.0;
  pdl_wait();
  double acc[kTile][kTile];
#pragma unroll
  for (int i = 0; i < kTile; ++i)
#pragma unroll
    for (int j = 0; j < kTile; ++j) acc[i][j] = 0.0;
  for (long long ks = k0; ks < k0 + kChunk; ks += kSlab) {
    // rows 0..99: 4 consecutive elements of one tangent row per item, hi (and lo) planes
    for (int e = tid; e < kLat * (kSlab / 4); e += kGramThreads) {
      const int row = e / (kSlab / 4), c4 = (e % (kSlab / 4)) * 4;
      const long long i = row * M + ks + c4;
      const uint2 hv = *reinterpret_cast<const uint2*>(tp + i);
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&hv);
      double v[4] = {(double)__low2float(h2[0]), (double)__high2float(h2[0]), (double)__low2float(h2[1]),
                     (double)__high2float(h2[1])};
      if (passes != 1) {
        const uint2 lv = *reinterpret_cast<const uint2*>(tp + plane + i);
        const __nv_bfloat162* l2 = reinterpret_cast<const __nv_bfloat162*>(&lv);
        v[0] += (double)__low2float(l2[0]);
        v[1] += (double)__high2float(l2[0]);
        v[2] += (double)__low2float(l2[1]);
        v[3] += (double)__high2float(l2[1]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) s[c4 + j][row] = v[j];
    }
    if (tid < kSlab) s[tid][kLat] = (double)cur[ks + tid] - (double)tgt[ks + tid];
    __syncthreads();
    if (live) {
#pragma unroll 2
      for (int k = 0; k < kSlab; ++k) {
        double a[kTile], b[kTile];
#pragma unroll
        for (int i = 0; i < kTile; i += 2) {
          const double2 av = *reinterpret_cast<const double2*>(&s[k][ti * kTile + i]);
          const double2 bv = *reinterpret_cast<const double2*>(&s[k][tj * kTile + i]);
          a[i] = av.x; a[i + 1] = av.y;
          b[i] = bv.x; b[i + 1] = bv.y;
        }
#pragma unroll
        for (int i = 0; i < kTile; ++i)
#pragma unroll
          for (int j = 0; j < kTile; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
  if (!live) return;
  double* o = part + ((size_t)chunk * kTiles + tid) * kTile * kTile;
#pragma unroll
  for (int i = 0; i < kTile; ++i)
#pragma unroll
    for (int j = 0; j < kTile; ++j) o[i * kTile + j] = acc[i][j];
}

// one thread per (i, j) of the 101 x 101 Gram: (i, j) and (j, i) add the same partials in the same order.  pixel: A, g, e
// already hold the pixel Gram (launch_gn_gram), which enters as a * pixel + features.  feats == 0: no feature terms.
__global__ void __launch_bounds__(256) feat_gram_reduce_kernel(const double* __restrict__ part, FeatWeights c, int feats, int pixel,
                                                               double* __restrict__ A, double* __restrict__ g,
                                                               double* __restrict__ e) {
  pdl_trigger();
  pdl_wait();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (kLat + 1) * (kLat + 1)) return;
  const int i = idx / (kLat + 1), j = idx % (kLat + 1);
  const int lo = min(i, j), hi = max(i, j), bi = lo / kTile, bj = hi / kTile;
  const int tile = bi * kTB - bi * (bi - 1) / 2 + (bj - bi);
  const double* p = part + (size_t)tile * kTile * kTile + (lo % kTile) * kTile + hi % kTile;
  double s = 0.0;
#pragma unroll
  for (int l = 0; l < 4 && feats; ++l) {
    double sl = 0.0;
    for (int ch = chunk0(l); ch < chunk0(l + 1); ++ch) sl += p[(size_t)ch * kTiles * kTile * kTile];
    s = fma(c.c[l], sl, s);
  }
  double* out = nullptr;
  if (i < kLat && j < kLat) out = A + i * kLat + j;
  else if (i < kLat) out = g + i;
  else if (i == kLat && j == kLat && e) out = e;
  if (out) *out = pixel ? fma(c.a, *out, s) : s;
}

// one CTA per sample.  As gn_accept_kernel, on E = a |x_hat - x|^2 + sum_i c_i |g_i(x_hat) - g_i(x)|^2: the trial's
// features are the plan's planes (tr), the target's and the current ones float32 NHWC (tgt, cur).  a == 0 leaves the
// pixels out (x is not read); feats == 0 the features (f is not read).
__global__ void __launch_bounds__(256) feat_accept_kernel(int init, const float* __restrict__ xht, const float* __restrict__ x,
                                                          FeatLayers f, FeatWeights c, int feats, int passes, float* xh,
                                                          double* __restrict__ e, double* __restrict__ lam,
                                                          float* __restrict__ z, const float* __restrict__ zt,
                                                          const int* __restrict__ ok, float* __restrict__ loss, long long ldl,
                                                          int col) {
  pdl_trigger();
  pdl_wait();
  __shared__ double red[256], redf[256];
  __shared__ int acc;
  const int k = blockIdx.x, t = threadIdx.x;
  const float* a = xht + (size_t)k * kPix;
  const float* b = x + (size_t)k * kPix;
  double s = 0.0, sf = 0.0;
  if (c.a != 0.0)
    for (int p = t; p < kPix; p += 256) {
      const double d = (double)a[p] - (double)b[p];
      s = fma(d, d, s);
    }
#pragma unroll
  for (int l = 0; l < 4 && feats; ++l) {
    const long long M = feat_m(l), base = (long long)k * M;
    double sl = 0.0;
    for (long long m = t; m < M; m += 256) {
      const double d = (double)plane_value(f.tan[l], f.plane[l], passes, base + m) - (double)f.tgt[l][base + m];
      sl = fma(d, d, sl);
    }
    sf = fma(c.c[l], sl, sf);
  }
  red[t] = s;
  redf[t] = sf;
  __syncthreads();
  for (int half = 128; half > 0; half >>= 1) {
    if (t < half) {
      red[t] += red[t + half];
      redf[t] += redf[t + half];
    }
    __syncthreads();
  }
  if (t == 0) {
    const double et = c.a != 0.0 ? fma(c.a, red[0], redf[0]) : redf[0];
    acc = gn_decide(init, et, ok, e, lam, loss, ldl, col, k) || init;
  }
  __syncthreads();
  if (!acc) return;
#pragma unroll
  for (int l = 0; l < 4 && feats; ++l) {
    const long long M = feat_m(l), base = (long long)k * M;
    for (long long m = t; m < M; m += 256) f.cur[l][base + m] = plane_value(f.tan[l], f.plane[l], passes, base + m);
  }
  if (init) return;
  for (int p = t; p < kPix; p += 256) xh[(size_t)k * kPix + p] = a[p];
  if (t < kLat) z[(size_t)k * kLat + t] = zt[(size_t)k * kLat + t];
}

// The deepest layer's value is what its backward GEMM's epilogue would write from a zero accumulator with the cotangent as
// `res`: (0 + res) * scale * lrelu'(a), res read as the GEMM reads it (hi + lo, or hi in bf16 mode), and it writes the
// planes that GEMM writes (in bf16 mode the lo plane only under a split-K finalize).  So a zero cotangent above it gives
// the same bits as leaving that layer out, and the encoder VJP's planes hold afterwards what its own GEMM leaves there.
// grid (tiles of the supplied layers, n), kCotThreads.  A tile is kCotCh channels x kCotPix pixels of one image and layer;
// layer l's tiles start at tile0.{x,y,z} for l = 1, 2, 3 (0 for l = 0).  The NCHW rows are read along pixels and the NHWC
// planes written along channels, both coalesced, through a padded shared-memory tile.
constexpr int kCotCh = 32, kCotPix = 16, kCotThreads = 128;
constexpr int cot_tiles(int l) { return ((128 << l) / kCotCh) * ((1024 >> (2 * l)) / kCotPix); }   // 256, 128, 64, 32

__global__ void __launch_bounds__(kCotThreads) feat_cotangent_kernel(FeatCotangents c, int passes, int3 tile0) {
  pdl_trigger();
  __shared__ float s[kCotCh][kCotPix + 1];
  const int t = blockIdx.x, k = blockIdx.y, tid = threadIdx.x;
  const int l = t >= tile0.z ? 3 : t >= tile0.y ? 2 : t >= tile0.x ? 1 : 0;
  const int C = 128 << l, HW = 1024 >> (2 * l);
  const int tt = t - (l == 3 ? tile0.z : l == 2 ? tile0.y : l == 1 ? tile0.x : 0);
  const int ch0 = tt / (HW / kCotPix) * kCotCh, px0 = tt % (HW / kCotPix) * kCotPix;
  const float* src = pick(c.c, l);
  __nv_bfloat16* dst = pick(c.out, l);
  const long long plane = pick(c.plane, l);
  pdl_wait();
#pragma unroll
  for (int i = 0; i < kCotCh * kCotPix / kCotThreads; ++i) {
    const int ch = tid / kCotPix + i * (kCotThreads / kCotPix), px = tid % kCotPix;
    s[ch][px] = src[((long long)k * C + ch0 + ch) * HW + px0 + px];
  }
  __syncthreads();
  const bool deep = l == c.deep;
  const int ch = tid % kCotCh;
  const float sc = deep && c.scale ? c.scale[ch0 + ch] : 1.f;
#pragma unroll
  for (int i = 0; i < kCotCh * kCotPix / kCotThreads; ++i) {
    const int px = tid / kCotCh + i * (kCotThreads / kCotCh);
    const long long o = ((long long)k * HW + px0 + px) * C + ch0 + ch;
    float v = s[ch][px];
    __nv_bfloat16 hi, lo;
    split_bf16(v, hi, lo);
    if (deep) {   // tapgemm's res + ACT_MASK epilogue on a zero accumulator: res as the GEMM reads it, then scale and mask
      const float r = passes == 1 ? __bfloat162float(hi) : __bfloat162float(hi) + __bfloat162float(lo);
      split_bf16(r * sc * (__bfloat162float(c.mask[o]) > 0.f ? 1.f : 0.2f), hi, lo);
    }
    dst[o] = hi;
    if (!deep || c.deep_lo) dst[plane + o] = lo;
  }
}

}  // namespace

size_t feat_part_doubles() { return (size_t)kChunks * kTiles * kTile * kTile; }

int launch_feat_store(const __nv_bfloat16* p, long long plane, int passes, int layer, int n, float* out, int nchw,
                      cudaStream_t st) {
  const long long total = (long long)n * feat_m(layer);
  const int blocks = (int)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096);
  if (launch_pdl(feat_store_kernel, dim3(blocks), dim3(256), 0, st, p, plane, passes, 128 << layer, 1024 >> (2 * layer), total,
                 out, nchw) != cudaSuccess)
    return -1;
  return 1;
}

int launch_feat_gram(const FeatLayers& t, const FeatWeights& c, int feats, int passes, int pixel, double* part, double* A,
                     double* g, double* e, cudaStream_t st) {
  if (feats && launch_pdl(feat_gram_kernel, dim3(kChunks), dim3(kGramThreads), 0, st, t, passes, part) != cudaSuccess)
    return -1;
  if (launch_pdl(feat_gram_reduce_kernel, dim3(((kLat + 1) * (kLat + 1) + 255) / 256), dim3(256), 0, st, (const double*)part, c,
                 feats, pixel, A, g, e) != cudaSuccess)
    return -1;
  return feats ? 2 : 1;
}

int launch_feat_accept(int init, const float* xht, const float* x, const FeatLayers& f, const FeatWeights& c, int feats,
                       int passes, float* xh, double* e, double* lam, float* z, const float* zt, const int* ok, float* loss,
                       long long ldl, int col, int n, cudaStream_t st) {
  if (launch_pdl(feat_accept_kernel, dim3(n), dim3(256), 0, st, init, xht, x, f, c, feats, passes, xh, e, lam, z, zt, ok, loss, ldl,
                 col) != cudaSuccess)
    return -1;
  return 1;
}

int launch_feat_cotangent(const FeatCotangents& c, int passes, int n, cudaStream_t st) {
  int first[5] = {0, 0, 0, 0, 0};
  for (int l = 0; l < 4; ++l) first[l + 1] = first[l] + (c.c[l] ? cot_tiles(l) : 0);
  if (first[4] == 0 || n == 0) return 0;
  if (launch_pdl(feat_cotangent_kernel, dim3(first[4], n), dim3(kCotThreads), 0, st, c, passes, make_int3(first[1], first[2], first[3])) !=
      cudaSuccess)
    return -1;
  return 1;
}

}  // namespace ian
