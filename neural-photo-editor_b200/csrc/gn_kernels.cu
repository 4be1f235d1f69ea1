// gn_kernels.cu -- the kernels of the latent fit (ian_decode_gauss_newton_*, ian_fit_latent_*; DESIGN section 5.6i).
// Per sample, with J the decoder's Jacobian at z as 100 rows of 12288 pixels (decode_jvp's output with the identity as
// tangents) and r = x_hat - x:
//   gn_replicate     : z -> the 100 x 100 batch of the Jacobian's JVP pass (every row z)
//   gn_gram          : partial sums of the upper triangle of [J | r]^T [J | r] over 16 pixel chunks, float64
//   gn_gram_reduce   : the chunk partials added in chunk order -> A = J^T J (both triangles), g = J^T r, e = r^T r
//   gn_solve         : Levenberg-Marquardt step: Cholesky of A + lambda D in float64, delta = -(A + lambda D)^-1 g,
//                      z_trial = float32(z + delta), or a rejected step when a pivot is not positive
//   gn_accept        : e_trial = |x_hat(z_trial) - x|^2 in a fixed order; accept / reject, lambda, the loss history
// Operands are float32; every product is formed in float64, where a product of two float32 values is exact, so A, g and e
// differ from a float64 Gram of the same J and r only by summation order.
// The masked fit under the prior (ian_map_gauss_newton_*, ian_fit_latent_map_*; DESIGN section 5.6j) runs the same bodies
// with a pixel weight w and a prior weight beta: map_gram weights one factor of every product by w (exact in float64),
// map_gram_reduce adds beta I, beta u and beta |u|^2 after the chunk sums, and map_accept reduces
// sum_p w_p (x_hat_p - x_p)^2 + beta |u|^2.  Pixels with w_p == 0 are staged or summed as nothing at all, so x there may
// hold anything, NaN included.  The unweighted kernels instantiate the bodies without a weight.
// The robust fit (ian_robust_gauss_newton_*, ian_fit_latent_robust_*; DESIGN section 5.6m) is iteratively reweighted least
// squares on E(u) = sum_p w_p rho(r_p^2) + beta |u|^2 with a per-sample scale delta (Huber or Cauchy rho): robust_gram runs
// gram_body with omega_p = w_p rho'(d^2) in place of w_p (then map_gram_reduce), robust_accept reduces the true E, and
// robust_scale picks delta from the lower median of |r| over the weighted pixels.  Where rho'(s) = 1 (Huber's quadratic
// region) omega_p is w_p itself, so Huber with delta = +inf stages map_gram's operands and sums map_accept's terms.
#include "edge.h"

namespace ian {

namespace {

constexpr int kPix = 12288;             // 3 x 64 x 64
constexpr int kLat = 100;
constexpr int kBlk = 32;                // the Gram's output blocks are 32 x 32
constexpr int kNBlk = 4;                // ceil(101 / 32): rows 0..99 are J, row 100 is r, the rest zero
constexpr int kPairs = kNBlk * (kNBlk + 1) / 2;   // blocks (bi <= bj) of the upper triangle
constexpr int kChunks = 16;             // pixel chunks per sample: kPairs x kChunks = 160 CTAs
constexpr int kChunkPix = kPix / kChunks;
constexpr int kSub = 64;                // pixels staged in shared memory per step
constexpr int kLd = kLat + 1;           // row stride of the solver's matrix in shared memory

// rho'(s) and rho(s) of the robust losses at s = d^2 (kind: IAN_ROBUST_HUBER / IAN_ROBUST_CAUCHY, dl the scale delta)
__device__ __forceinline__ double robust_dw(int kind, double dl, double s) {
  if (kind == kRobustHuber) return s <= dl * dl ? 1.0 : dl / sqrt(s);
  return 1.0 / (1.0 + s / (dl * dl));
}

// s + wp rho(d^2), with Huber's quadratic region summed exactly as map_accept sums every pixel
__device__ __forceinline__ double robust_add(int kind, double dl, double wp, double d, double s) {
  const double q = d * d, d2 = dl * dl;
  if (kind == kRobustHuber) return q <= d2 ? fma(wp * d, d, s) : fma(wp, 2.0 * dl * fabs(d) - d2, s);
  return fma(wp, d2 * log1p(q / d2), s);
}

__device__ __forceinline__ double gram_row(const float* __restrict__ J, const float* __restrict__ xh,
                                           const float* __restrict__ x, int row, int p) {
  if (row < kLat) return (double)J[(size_t)row * kPix + p];
  if (row == kLat) return (double)xh[p] - (double)x[p];
  return 0.0;
}

__global__ void __launch_bounds__(256) gn_replicate_kernel(const float* __restrict__ z, float* __restrict__ zrep) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kLat * kLat) zrep[i] = z[i % kLat];
}

// grid (kPairs, kChunks), 256 threads, each a 2 x 2 tile of the 32 x 32 output block; part[chunk][pair][32][32].
// kMap: w (nullable: all ones) multiplies the first factor of every product; a pixel with w == 0 stages zeros in both.
// kRobust: omega = w rho'(d^2) at the sample's scale *dl does, in its place; omega == 0 stages zeros.  Thread t stages only
// pixel p0 + t % kSub (256 is a multiple of kSub), so it forms that pixel's omega once per step.
template <bool kMap, bool kRobust = false>
__device__ __forceinline__ void gram_body(const float* __restrict__ J, const float* __restrict__ xh,
                                          const float* __restrict__ x, const float* __restrict__ w, double* __restrict__ part,
                                          int kind = 0, const double* __restrict__ dl = nullptr) {
  pdl_trigger();
  pdl_wait();
  __shared__ double sa[kSub][kBlk + 1], sb[kSub][kBlk + 1];
  int q = blockIdx.x, bi = 0;
  while (q >= kNBlk - bi) { q -= kNBlk - bi; ++bi; }
  const int bj = bi + q, chunk = blockIdx.y, t = threadIdx.x;
  const int ti = (t >> 4) * 2, tj = (t & 15) * 2;
  double acc00 = 0.0, acc01 = 0.0, acc10 = 0.0, acc11 = 0.0;
  for (int p0 = chunk * kChunkPix; p0 < (chunk + 1) * kChunkPix; p0 += kSub) {
    double om = 0.0;
    if constexpr (kRobust) {
      const int p = p0 + t % kSub;
      const double wp = w ? (double)w[p] : 1.0, d = (double)xh[p] - (double)x[p];
      om = wp == 0.0 ? 0.0 : wp * robust_dw(kind, *dl, d * d);
    }
    for (int e = t; e < kBlk * kSub; e += 256) {
      const int r = e / kSub, p = e % kSub;
      if (kRobust) {
        sa[p][r] = om == 0.0 ? 0.0 : om * gram_row(J, xh, x, bi * kBlk + r, p0 + p);
        sb[p][r] = om == 0.0 ? 0.0 : gram_row(J, xh, x, bj * kBlk + r, p0 + p);
      } else if (kMap && w) {
        const double wp = (double)w[p0 + p];
        sa[p][r] = wp == 0.0 ? 0.0 : wp * gram_row(J, xh, x, bi * kBlk + r, p0 + p);
        sb[p][r] = wp == 0.0 ? 0.0 : gram_row(J, xh, x, bj * kBlk + r, p0 + p);
      } else {
        sa[p][r] = gram_row(J, xh, x, bi * kBlk + r, p0 + p);
        sb[p][r] = gram_row(J, xh, x, bj * kBlk + r, p0 + p);
      }
    }
    __syncthreads();
#pragma unroll 8
    for (int p = 0; p < kSub; ++p) {
      const double a0 = sa[p][ti], a1 = sa[p][ti + 1], b0 = sb[p][tj], b1 = sb[p][tj + 1];
      acc00 = fma(a0, b0, acc00);
      acc01 = fma(a0, b1, acc01);
      acc10 = fma(a1, b0, acc10);
      acc11 = fma(a1, b1, acc11);
    }
    __syncthreads();
  }
  double* o = part + ((size_t)(chunk * kPairs + blockIdx.x) * kBlk + ti) * kBlk + tj;
  o[0] = acc00;
  o[1] = acc01;
  o[kBlk] = acc10;
  o[kBlk + 1] = acc11;
}

__global__ void __launch_bounds__(256) gn_gram_kernel(const float* __restrict__ J, const float* __restrict__ xh,
                                                      const float* __restrict__ x, double* __restrict__ part) {
  gram_body<false>(J, xh, x, nullptr, part);
}

__global__ void __launch_bounds__(256) map_gram_kernel(const float* __restrict__ J, const float* __restrict__ xh,
                                                       const float* __restrict__ x, const float* __restrict__ w,
                                                       double* __restrict__ part) {
  gram_body<true>(J, xh, x, w, part);
}

__global__ void __launch_bounds__(256) robust_gram_kernel(const float* __restrict__ J, const float* __restrict__ xh,
                                                          const float* __restrict__ x, const float* __restrict__ w, int kind,
                                                          const double* __restrict__ dl, double* __restrict__ part) {
  gram_body<true, true>(J, xh, x, w, part, kind, dl);
}

// beta |u|^2 of one sample's float32 u (100), in one fixed order
__device__ __forceinline__ double prior_sq(const float* __restrict__ u) {
  double s = 0.0;
  for (int i = 0; i < kLat; ++i) s = fma((double)u[i], (double)u[i], s);
  return s;
}

// one thread per (i, j) of the 101 x 101 Gram: (i, j) and (j, i) add the same partials in the same order, so A is exactly
// symmetric.  kMap: then A_ii += beta, g_i += beta u_i, e += beta |u|^2, each added once.
template <bool kMap>
__device__ __forceinline__ void gram_reduce_body(const double* __restrict__ part, double beta, const float* __restrict__ u,
                                                 double* __restrict__ A, double* __restrict__ g, double* __restrict__ e) {
  pdl_trigger();
  pdl_wait();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (kLat + 1) * (kLat + 1)) return;
  const int i = idx / (kLat + 1), j = idx % (kLat + 1);
  const int lo = min(i, j), hi = max(i, j), bi = lo / kBlk, bj = hi / kBlk;
  const int pair = bi * kNBlk - bi * (bi - 1) / 2 + (bj - bi);
  const double* p = part + ((size_t)pair * kBlk + lo % kBlk) * kBlk + hi % kBlk;
  double s = 0.0;
  for (int c = 0; c < kChunks; ++c) s += p[(size_t)c * kPairs * kBlk * kBlk];
  if (i < kLat && j < kLat) A[i * kLat + j] = kMap && i == j ? s + beta : s;
  else if (i < kLat) g[i] = kMap ? fma(beta, (double)u[i], s) : s;
  else if (i == kLat && j == kLat && e) *e = kMap ? fma(beta, prior_sq(u), s) : s;
}

__global__ void __launch_bounds__(256) gn_gram_reduce_kernel(const double* __restrict__ part, double* __restrict__ A,
                                                             double* __restrict__ g, double* __restrict__ e) {
  gram_reduce_body<false>(part, 0.0, nullptr, A, g, e);
}

__global__ void __launch_bounds__(256) map_gram_reduce_kernel(const double* __restrict__ part, double beta,
                                                              const float* __restrict__ u, double* __restrict__ A,
                                                              double* __restrict__ g, double* __restrict__ e) {
  gram_reduce_body<true>(part, beta, u, A, g, e);
}

// one CTA per sample; dynamic shared memory: the 100 x kLd float64 matrix
__global__ void __launch_bounds__(256) gn_solve_kernel(const double* __restrict__ A, const double* __restrict__ g,
                                                       const double* __restrict__ lam, const float* __restrict__ z,
                                                       float* __restrict__ zt, int* __restrict__ ok) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ double M[];
  __shared__ double b[kLat];
  __shared__ double dmax;
  __shared__ int bad;
  const int k = blockIdx.x, t = threadIdx.x;
  const double* Ak = A + (size_t)k * kLat * kLat;
  if (t == 0) {
    double m = 0.0;
    for (int i = 0; i < kLat; ++i) m = fmax(m, Ak[i * (kLat + 1)]);
    dmax = m;
    bad = 0;
  }
  __syncthreads();
  const double l = lam[k], dfloor = kGnDampFloor * dmax;
  for (int e = t; e < kLat * kLat; e += 256) {
    const int i = e / kLat, j = e % kLat;
    double v = Ak[e];
    if (i == j) v += l * fmax(v, dfloor);
    M[i * kLd + j] = v;
  }
  for (int i = t; i < kLat; i += 256) b[i] = -g[(size_t)k * kLat + i];
  __syncthreads();
  // Cholesky M = L L^T, right-looking, L in the lower triangle; every element is updated by one thread in column order
  for (int c = 0; c < kLat; ++c) {
    if (t == 0) {
      const double d = M[c * kLd + c];
      if (!(d > 0.0)) bad = 1;                            // also NaN
      M[c * kLd + c] = sqrt(d);
    }
    __syncthreads();
    if (bad) break;
    const double dc = M[c * kLd + c];
    for (int i = c + 1 + t; i < kLat; i += 256) M[i * kLd + c] /= dc;
    __syncthreads();
    const int m = kLat - 1 - c;
    for (int e = t; e < m * m; e += 256) {
      const int i = c + 1 + e / m, j = c + 1 + e % m;
      if (j <= i) M[i * kLd + j] = fma(-M[i * kLd + c], M[j * kLd + c], M[i * kLd + j]);
    }
    __syncthreads();
  }
  if (!bad) {
    for (int c = 0; c < kLat; ++c) {                      // L y = -g
      if (t == 0) b[c] /= M[c * kLd + c];
      __syncthreads();
      for (int i = c + 1 + t; i < kLat; i += 256) b[i] = fma(-M[i * kLd + c], b[c], b[i]);
      __syncthreads();
    }
    for (int c = kLat - 1; c >= 0; --c) {                 // L^T delta = y
      if (t == 0) b[c] /= M[c * kLd + c];
      __syncthreads();
      for (int i = t; i < c; i += 256) b[i] = fma(-M[c * kLd + i], b[c], b[i]);
      __syncthreads();
    }
  }
  float v = 0.f;
  int fin = 1;
  if (t < kLat) {
    v = z[(size_t)k * kLat + t];
    if (!bad) {
      const float w = (float)((double)v + b[t]);
      fin = isfinite(w);
      v = w;
    }
  }
  const int good = !bad && __syncthreads_and(fin);
  if (t < kLat) zt[(size_t)k * kLat + t] = good ? v : z[(size_t)k * kLat + t];
  if (t == 0) ok[k] = good;
}

// one CTA per sample.  init: x_hat_trial is the start's decode (x_hat itself).  e_trial, then gn_decide (edge.h); a taken
// step also copies z <- z_trial, x_hat <- x_hat_trial.
// kMap: e_trial = sum over w != 0 of w (x_hat_trial - x)^2 (w nullable: all ones) + beta |z_trial|^2 (init: |z|^2).
// kRobust: sum over w != 0 of w rho((x_hat_trial - x)^2) at the sample's scale dl[k] instead, in the same order.
template <bool kMap, bool kRobust = false>
__device__ __forceinline__ void accept_body(int init, const float* __restrict__ xht, const float* __restrict__ x,
                                            const float* __restrict__ w, double beta, float* xh, double* __restrict__ e,
                                            double* __restrict__ lam, float* __restrict__ z, const float* __restrict__ zt,
                                            const int* __restrict__ ok, float* __restrict__ loss, long long ldl, int col,
                                            int kind = 0, const double* __restrict__ dl = nullptr) {
  pdl_trigger();
  pdl_wait();
  __shared__ double red[256];
  __shared__ int acc;
  const int k = blockIdx.x, t = threadIdx.x;
  const float* a = xht + (size_t)k * kPix;
  const float* b = x + (size_t)k * kPix;
  const float* wk = kMap && w ? w + (size_t)k * kPix : nullptr;
  double s = 0.0;
  const double dk = kRobust ? dl[k] : 0.0;
  for (int p = t; p < kPix; p += 256) {
    if (kRobust) {
      const double wp = wk ? (double)wk[p] : 1.0;
      if (wp == 0.0) continue;
      s = robust_add(kind, dk, wp, (double)a[p] - (double)b[p], s);
    } else if (kMap && wk) {
      const double wp = (double)wk[p];
      if (wp == 0.0) continue;
      const double d = (double)a[p] - (double)b[p];
      s = fma(wp * d, d, s);
    } else {
      const double d = (double)a[p] - (double)b[p];
      s = fma(d, d, s);
    }
  }
  red[t] = s;
  __syncthreads();
  for (int half = 128; half > 0; half >>= 1) {
    if (t < half) red[t] += red[t + half];
    __syncthreads();
  }
  if (t == 0) {
    double et = red[0];
    if (kMap) et = fma(beta, prior_sq((init ? z : zt) + (size_t)k * kLat), et);
    acc = gn_decide(init, et, ok, e, lam, loss, ldl, col, k);
  }
  __syncthreads();
  if (!acc) return;
  for (int p = t; p < kPix; p += 256) xh[(size_t)k * kPix + p] = a[p];
  if (t < kLat) z[(size_t)k * kLat + t] = zt[(size_t)k * kLat + t];
}

__global__ void __launch_bounds__(256) gn_accept_kernel(int init, const float* __restrict__ xht, const float* __restrict__ x,
                                                        float* xh, double* __restrict__ e, double* __restrict__ lam,
                                                        float* __restrict__ z, const float* __restrict__ zt,
                                                        const int* __restrict__ ok, float* __restrict__ loss, long long ldl,
                                                        int col) {
  accept_body<false>(init, xht, x, nullptr, 0.0, xh, e, lam, z, zt, ok, loss, ldl, col);
}

__global__ void __launch_bounds__(256) map_accept_kernel(int init, const float* __restrict__ xht, const float* __restrict__ x,
                                                         const float* __restrict__ w, double beta, float* xh,
                                                         double* __restrict__ e, double* __restrict__ lam,
                                                         float* __restrict__ z, const float* __restrict__ zt,
                                                         const int* __restrict__ ok, float* __restrict__ loss, long long ldl,
                                                         int col) {
  accept_body<true>(init, xht, x, w, beta, xh, e, lam, z, zt, ok, loss, ldl, col);
}

__global__ void __launch_bounds__(256) robust_accept_kernel(int init, const float* __restrict__ xht,
                                                            const float* __restrict__ x, const float* __restrict__ w,
                                                            double beta, int kind, const double* __restrict__ dl, float* xh,
                                                            double* __restrict__ e, double* __restrict__ lam,
                                                            float* __restrict__ z, const float* __restrict__ zt,
                                                            const int* __restrict__ ok, float* __restrict__ loss,
                                                            long long ldl, int col) {
  accept_body<true, true>(init, xht, x, w, beta, xh, e, lam, z, zt, ok, loss, ldl, col, kind, dl);
}

// one CTA per sample: dl[k] = max(m c, kRobustScaleFloor), m the lower median (rank (count - 1) / 2) of float32 |x_hat - x|
// over the pixels with w != 0, selected exactly on the bit patterns (monotone for non-negative floats) by four 8-bit radix
// passes from the top byte; kRobustScaleFloor when no pixel is weighted.  The histograms count with shared-memory atomics,
// whose totals do not depend on their order.
__global__ void __launch_bounds__(256) robust_scale_kernel(const float* __restrict__ xh, const float* __restrict__ x,
                                                           const float* __restrict__ w, double c, double* __restrict__ dl) {
  pdl_trigger();
  pdl_wait();
  __shared__ unsigned hist[256];
  __shared__ unsigned cnt, prefix, rank;
  const int k = blockIdx.x, t = threadIdx.x;
  const float* a = xh + (size_t)k * kPix;
  const float* b = x + (size_t)k * kPix;
  const float* wk = w ? w + (size_t)k * kPix : nullptr;
  if (t == 0) cnt = prefix = 0;
  __syncthreads();
  unsigned mine = 0;
  for (int p = t; p < kPix; p += 256) mine += !wk || wk[p] != 0.f;
  atomicAdd(&cnt, mine);
  __syncthreads();
  if (cnt == 0) {
    if (t == 0) dl[k] = kRobustScaleFloor;
    return;
  }
  if (t == 0) rank = (cnt - 1) / 2;
  unsigned mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    hist[t] = 0;
    __syncthreads();
    const unsigned pre = prefix;
    for (int p = t; p < kPix; p += 256) {
      if (wk && wk[p] == 0.f) continue;
      const unsigned v = __float_as_uint(fabsf(a[p] - b[p]));
      if ((v & mask) == pre) atomicAdd(&hist[(v >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (t == 0) {
      unsigned below = 0, j = 0;
      while (below + hist[j] <= rank) below += hist[j++];
      rank -= below;
      prefix = pre | (j << shift);
    }
    mask |= 255u << shift;
    __syncthreads();
  }
  if (t == 0) dl[k] = fmax((double)__uint_as_float(prefix) * c, kRobustScaleFloor);
}

// out (n,12288) = rho'((x_hat - x)^2) at the sample's scale dl[k] as float32, 0 where w == 0
__global__ void __launch_bounds__(256) robust_outliers_kernel(const float* __restrict__ xh, const float* __restrict__ x,
                                                              const float* __restrict__ w, int kind,
                                                              const double* __restrict__ dl, float* __restrict__ out,
                                                              long long total) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  if (w && w[i] == 0.f) {
    out[i] = 0.f;
    return;
  }
  const double d = (double)xh[i] - (double)x[i];
  out[i] = (float)robust_dw(kind, dl[i / kPix], d * d);
}

constexpr size_t kSolveSmem = (size_t)kLat * kLd * sizeof(double);

}  // namespace

size_t gn_part_doubles() { return (size_t)kChunks * kPairs * kBlk * kBlk; }

int launch_gn_replicate(const float* z, float* zrep, cudaStream_t st) {
  if (launch_pdl(gn_replicate_kernel, dim3((kLat * kLat + 255) / 256), dim3(256), 0, st, z, zrep) != cudaSuccess) return -1;
  return 1;
}

int launch_gn_gram(const float* J, const float* xh, const float* x, double* part, double* A, double* g, double* e,
                   cudaStream_t st) {
  if (launch_pdl(gn_gram_kernel, dim3(kPairs, kChunks), dim3(256), 0, st, J, xh, x, part) != cudaSuccess) return -1;
  if (launch_pdl(gn_gram_reduce_kernel, dim3(((kLat + 1) * (kLat + 1) + 255) / 256), dim3(256), 0, st, (const double*)part, A,
                 g, e) != cudaSuccess)
    return -1;
  return 2;
}

int launch_map_gram(const float* J, const float* xh, const float* x, const float* w, double beta, const float* u, double* part,
                    double* A, double* g, double* e, cudaStream_t st) {
  if (launch_pdl(map_gram_kernel, dim3(kPairs, kChunks), dim3(256), 0, st, J, xh, x, w, part) != cudaSuccess) return -1;
  if (launch_pdl(map_gram_reduce_kernel, dim3(((kLat + 1) * (kLat + 1) + 255) / 256), dim3(256), 0, st, (const double*)part,
                 beta, u, A, g, e) != cudaSuccess)
    return -1;
  return 2;
}

int launch_robust_gram(const float* J, const float* xh, const float* x, const float* w, int kind, const double* dl, double beta,
                       const float* u, double* part, double* A, double* g, cudaStream_t st) {
  if (launch_pdl(robust_gram_kernel, dim3(kPairs, kChunks), dim3(256), 0, st, J, xh, x, w, kind, dl, part) != cudaSuccess)
    return -1;
  if (launch_pdl(map_gram_reduce_kernel, dim3(((kLat + 1) * (kLat + 1) + 255) / 256), dim3(256), 0, st, (const double*)part,
                 beta, u, A, g, (double*)nullptr) != cudaSuccess)
    return -1;
  return 2;
}

int launch_robust_scale(const float* xh, const float* x, const float* w, int kind, double* dl, int n, cudaStream_t st) {
  const double c = kind == kRobustHuber ? kRobustHuberC : kRobustCauchyC;
  if (launch_pdl(robust_scale_kernel, dim3(n), dim3(256), 0, st, xh, x, w, c, dl) != cudaSuccess) return -1;
  return 1;
}

int launch_robust_outliers(const float* xh, const float* x, const float* w, int kind, const double* dl, float* out, int n,
                           cudaStream_t st) {
  const long long total = (long long)n * kPix;
  if (launch_pdl(robust_outliers_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, xh, x, w, kind, dl, out,
                 total) != cudaSuccess)
    return -1;
  return 1;
}

int launch_gn_solve(const double* A, const double* g, const double* lam, const float* z, float* zt, int* ok, int n,
                    cudaStream_t st) {
  static DeviceOnce attr_set;
  const int dev = cur_device();
  if (!attr_set.is_done(dev)) {
    if (cudaFuncSetAttribute(gn_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSolveSmem) != cudaSuccess)
      return -1;
    attr_set.set_done(dev);
  }
  if (launch_pdl(gn_solve_kernel, dim3(n), dim3(256), kSolveSmem, st, A, g, lam, z, zt, ok) != cudaSuccess) return -1;
  return 1;
}

int launch_gn_accept(int init, const float* xht, const float* x, float* xh, double* e, double* lam, float* z, const float* zt,
                     const int* ok, float* loss, long long ldl, int col, int n, cudaStream_t st) {
  if (launch_pdl(gn_accept_kernel, dim3(n), dim3(256), 0, st, init, xht, x, xh, e, lam, z, zt, ok, loss, ldl, col) != cudaSuccess)
    return -1;
  return 1;
}

int launch_map_accept(int init, const float* xht, const float* x, const float* w, double beta, float* xh, double* e, double* lam,
                      float* u, const float* ut, const int* ok, float* loss, long long ldl, int col, int n, cudaStream_t st) {
  if (launch_pdl(map_accept_kernel, dim3(n), dim3(256), 0, st, init, xht, x, w, beta, xh, e, lam, u, ut, ok, loss, ldl, col) !=
      cudaSuccess)
    return -1;
  return 1;
}

int launch_robust_accept(int init, const float* xht, const float* x, const float* w, double beta, int kind, const double* dl,
                         float* xh, double* e, double* lam, float* u, const float* ut, const int* ok, float* loss, long long ldl,
                         int col, int n, cudaStream_t st) {
  if (launch_pdl(robust_accept_kernel, dim3(n), dim3(256), 0, st, init, xht, x, w, beta, kind, dl, xh, e, lam, u, ut, ok, loss,
                 ldl, col) != cudaSuccess)
    return -1;
  return 1;
}

}  // namespace ian
