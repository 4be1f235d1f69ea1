// train_kernels.cu -- the training-mode pieces that sit next to the hot path (SURVEY.md 8(f) rank 4).  The trainers
// (train_IAN*.py) stay the reference's; these are the two forward ops of the graphs that differ between
// `deterministic=True` (what API.IAN compiles, everything else in this library) and training mode:
//
//   * BatchNorm with BATCH statistics -- lasagne BatchNormLayer.get_output_for(deterministic=False), which every
//     `BN(...)` of IAN_simple.py:84-170 / IAN.py / layers.py:411-416 becomes in training:
//         mean = x.mean(axes), inv_std = 1/sqrt(x.var(axes) + eps)         (axes = all but the channel axis; biased var)
//         y = (x - mean) * (gamma * inv_std) + beta
//         running_mean    <- (1-alpha) running_mean    + alpha mean        (alpha = 0.1, eps = 1e-4: lasagne defaults)
//         running_inv_std <- (1-alpha) running_inv_std + alpha inv_std
//     Split in two calls so that data-parallel ranks can all-reduce (sum, sumsq) in between: cross-GPU synchronised BN.
//     The reductions use warp shuffles (north_star) and a fixed two-level order: bit-reproducible, no atomics.
//     Every partial sum is float64 from the first term, so Σx / Σx² lose only float64 roundings; the variance
//     Σx²/N - mean² then cancels them to a relative error of about 1e-16 (|mean| / std)², far below float32.
//   * MinibatchLayer (reference layers.py:486-524), the minibatch-discrimination features of the discriminator head.
#include <cuda_runtime.h>
#include <stdint.h>

namespace ian {

namespace {

constexpr int kBnSplits = 32;      // CTAs per channel (conv-shaped inputs); partial sums are added in split order

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum of (a, b): shuffles inside each warp, one smem slot per warp, first warp adds the slots in order
__device__ __forceinline__ void block_sum2(double& a, double& b) {
  __shared__ double sa[32], sb[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  a = warp_sum(a);
  b = warp_sum(b);
  if (lane == 0) { sa[warp] = a; sb[warp] = b; }
  __syncthreads();
  if (warp == 0) {
    a = lane < nw ? sa[lane] : 0.0;
    b = lane < nw ? sb[lane] : 0.0;
    a = warp_sum(a);
    b = warp_sum(b);
  }
}

// x: (n, c, hw) float32.  CTA (ch, split) reduces images [split*n/S, (split+1)*n/S) of channel ch.
__global__ void __launch_bounds__(256) bn_partial_kernel(const float* __restrict__ x, int n, int c, int hw,
                                                         double* __restrict__ part /*[c][S][2]*/) {
  const int ch = blockIdx.x, sp = blockIdx.y, S = gridDim.y;
  const int i0 = (int)((long long)n * sp / S), i1 = (int)((long long)n * (sp + 1) / S);
  double s = 0.0, q = 0.0;                               // float64 from the first term: v*v of a float32 v is exact
  for (int i = i0; i < i1; ++i) {
    const float* row = x + ((long long)i * c + ch) * hw;
    for (int k = threadIdx.x; k < hw; k += blockDim.x) {
      const double v = (double)__ldg(row + k);
      s += v;
      q += v * v;
    }
  }
  block_sum2(s, q);
  if (threadIdx.x == 0) {
    part[((long long)ch * S + sp) * 2] = s;
    part[((long long)ch * S + sp) * 2 + 1] = q;
  }
}

// dense inputs (hw == 1): x (n, c); one thread per channel (coalesced over channels), rows in order
__global__ void __launch_bounds__(256) bn_partial_dense_kernel(const float* __restrict__ x, int n, int c, double* __restrict__ part /*[c][S][2]*/) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x, sp = blockIdx.y, S = gridDim.y;
  if (ch >= c) return;
  const int i0 = (int)((long long)n * sp / S), i1 = (int)((long long)n * (sp + 1) / S);
  double s = 0.0, q = 0.0;
  for (int i = i0; i < i1; ++i) {
    const double v = (double)__ldg(x + (long long)i * c + ch);
    s += v;
    q += v * v;
  }
  part[((long long)ch * S + sp) * 2] = s;
  part[((long long)ch * S + sp) * 2 + 1] = q;
}

__global__ void bn_reduce_kernel(const double* __restrict__ part, int c, int S, double* __restrict__ sum, double* __restrict__ sumsq) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  double s = 0.0, q = 0.0;
  for (int k = 0; k < S; ++k) {                          // fixed order
    s += part[((long long)ch * S + k) * 2];
    q += part[((long long)ch * S + k) * 2 + 1];
  }
  sum[ch] = s;
  sumsq[ch] = q;
}

// per channel: statistics from the (possibly all-reduced) sums, running-average update, folded scale/shift
__global__ void bn_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ sumsq, double count, int c,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float alpha,
                                   float* __restrict__ running_mean, float* __restrict__ running_inv_std,
                                   float* __restrict__ scale_shift /*[2][c]*/) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  const double mean = sum[ch] / count;
  double var = sumsq[ch] / count - mean * mean;          // biased variance, as theano's x.var(axes)
  if (var < 0.0) var = 0.0;
  const float mean_f = (float)mean;
  const float inv_std = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean) running_mean[ch] = (1.f - alpha) * running_mean[ch] + alpha * mean_f;
  if (running_inv_std) running_inv_std[ch] = (1.f - alpha) * running_inv_std[ch] + alpha * inv_std;
  const float g = gamma ? gamma[ch] : 1.f, b = beta ? beta[ch] : 0.f;
  scale_shift[ch] = g * inv_std;
  scale_shift[c + ch] = mean_f;                          // y = (x - mean) * (gamma * inv_std) + beta, in lasagne's order
  scale_shift[2 * c + ch] = b;
}

__global__ void __launch_bounds__(256) bn_apply_kernel(const float* __restrict__ x, long long total, int c, int hw,
                                                       const float* __restrict__ ss /*[3][c]: scale, mean, beta*/, float* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)((i / hw) % c);
  y[i] = (x[i] - ss[c + ch]) * ss[ch] + ss[2 * c + ch];
}

// ---- MinibatchLayer (reference layers.py:486-524) ---------------------------------------------------------------
// W[d][k][p] = theta[d][k][p] * exp(lws[k][p]) / sqrt(sum_d theta[d][k][p]^2)                      (layers.py:495)
__global__ void __launch_bounds__(256) mb_colscale_kernel(const float* __restrict__ theta, const float* __restrict__ lws, int d, int kp,
                                                          float* __restrict__ colscale /*[kp]*/) {
  const int col = blockIdx.x;
  double s = 0.0, dummy = 0.0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    const double v = (double)__ldg(theta + (long long)i * kp + col);
    s += v * v;
  }
  block_sum2(s, dummy);
  if (threadIdx.x == 0) colscale[col] = (float)((double)expf(lws[col]) / sqrt(s));
}

// activation[i][col] = colscale[col] * sum_d x[i][d] * theta[d][col]   (T.tensordot(input, W, [[1],[0]]), layers.py:508)
// tile: 16 samples x 64 columns per CTA, d in chunks of 32 through shared memory
__global__ void __launch_bounds__(256) mb_activation_kernel(const float* __restrict__ x, const float* __restrict__ theta,
                                                            const float* __restrict__ colscale, int n, int d, int kp,
                                                            float* __restrict__ act /*[n][kp]*/) {
  __shared__ float Xs[16][33];
  __shared__ float Ts[32][65];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;     // 64 columns x 4 row groups (4 samples each)
  const int col0 = blockIdx.x * 64, i0 = blockIdx.y * 16;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int d0 = 0; d0 < d; d0 += 32) {
    for (int e = threadIdx.x; e < 16 * 32; e += 256) {
      const int r = e >> 5, k = e & 31;
      Xs[r][k] = (i0 + r < n && d0 + k < d) ? __ldg(x + (long long)(i0 + r) * d + d0 + k) : 0.f;
    }
    for (int e = threadIdx.x; e < 32 * 64; e += 256) {
      const int k = e >> 6, cc = e & 63;
      Ts[k][cc] = (d0 + k < d && col0 + cc < kp) ? __ldg(theta + (long long)(d0 + k) * kp + col0 + cc) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < 32; ++k) {
      const float t = Ts[k][tx];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(Xs[ty * 4 + j][k], t, acc[j]);
    }
    __syncthreads();
  }
  if (col0 + tx < kp)
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (i0 + ty * 4 + j < n) act[(long long)(i0 + ty * 4 + j) * kp + col0 + tx] = acc[j] * colscale[col0 + tx];
}

// f[i][k] = sum_j exp(-(sum_p |act[i,k,p] - act[j,k,p]| + 1e6 [i == j])) + b[k];  out = concat(x, f)   (layers.py:509-524)
__global__ void __launch_bounds__(128) mb_features_kernel(const float* __restrict__ x, const float* __restrict__ act, const float* __restrict__ b,
                                                          int n, int d, int K, int P, float* __restrict__ out /*[n][d+K]*/) {
  const int i = blockIdx.x;
  for (int e = threadIdx.x; e < d; e += blockDim.x) out[(long long)i * (d + K) + e] = x[(long long)i * d + e];
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float f = 0.f;
    for (int j = 0; j < n; ++j) {                        // fixed order
      float ad = (i == j) ? 1e6f : 0.f;
      for (int p = 0; p < P; ++p) ad += fabsf(act[(long long)i * K * P + k * P + p] - act[(long long)j * K * P + k * P + p]);
      f += expf(-ad);
    }
    out[(long long)i * (d + K) + d + k] = f + b[k];
  }
}

// ---- reverse mode (DESIGN §5.6b) ---------------------------------------------------------------------------------
// BatchNorm backward sums: CTA (ch, split) as bn_partial_kernel, Σdy and Σdy·x instead of Σx and Σx².  dy*x of two
// float32 values is exact in float64, and every partial is float64 from the first term.
__global__ void __launch_bounds__(256) bn_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy, int n, int c,
                                                             int hw, double* __restrict__ part /*[c][S][2]*/) {
  const int ch = blockIdx.x, sp = blockIdx.y, S = gridDim.y;
  const int i0 = (int)((long long)n * sp / S), i1 = (int)((long long)n * (sp + 1) / S);
  double s = 0.0, q = 0.0;
  for (int i = i0; i < i1; ++i) {
    const long long row = ((long long)i * c + ch) * hw;
    for (int k = threadIdx.x; k < hw; k += blockDim.x) {
      const double g = (double)__ldg(dy + row + k);
      s += g;
      q += g * (double)__ldg(x + row + k);
    }
  }
  block_sum2(s, q);
  if (threadIdx.x == 0) {
    part[((long long)ch * S + sp) * 2] = s;
    part[((long long)ch * S + sp) * 2 + 1] = q;
  }
}

__global__ void __launch_bounds__(256) bn_bwd_partial_dense_kernel(const float* __restrict__ x, const float* __restrict__ dy, int n, int c,
                                                                   double* __restrict__ part /*[c][S][2]*/) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x, sp = blockIdx.y, S = gridDim.y;
  if (ch >= c) return;
  const int i0 = (int)((long long)n * sp / S), i1 = (int)((long long)n * (sp + 1) / S);
  double s = 0.0, q = 0.0;
  for (int i = i0; i < i1; ++i) {
    const double g = (double)__ldg(dy + (long long)i * c + ch);
    s += g;
    q += g * (double)__ldg(x + (long long)i * c + ch);
  }
  part[((long long)ch * S + sp) * 2] = s;
  part[((long long)ch * S + sp) * 2 + 1] = q;
}

// mean and inv_std in float64 from the forward's sums, as bn_finalize_kernel forms them before its float32 roundings
__device__ __forceinline__ void bn_stats(const double* sum, const double* sumsq, double count, float eps, int ch, double& mean, double& s) {
  mean = sum[ch] / count;
  double var = sumsq[ch] / count - mean * mean;
  if (var < 0.0) var = 0.0;
  s = 1.0 / sqrt(var + (double)eps);
}

// this rank's dbeta = Σdy and dgamma = s (Σdy·x - mean Σdy) = Σ dy·x̂, both in float64 before the one rounding
__global__ void bn_bwd_params_kernel(const double* __restrict__ sum, const double* __restrict__ sumsq, double count, float eps,
                                     const double* __restrict__ sum_dy, const double* __restrict__ sum_dyx, int c,
                                     float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  double mean, s;
  bn_stats(sum, sumsq, count, eps, ch, mean, s);
  if (dgamma) dgamma[ch] = (float)(s * (sum_dyx[ch] - mean * sum_dy[ch]));
  if (dbeta) dbeta[ch] = (float)sum_dy[ch];
}

// dx = gamma s (dy - Σdy/N - x̂ Σ(dy x̂)/N) = a (dy - m - (x - mean) k), a = gamma s, m = Σdy/N, k = s² Σ(dy x̂)/N
__global__ void bn_bwd_coef_kernel(const double* __restrict__ sum, const double* __restrict__ sumsq, double count, float eps,
                                   const double* __restrict__ sum_dy, const double* __restrict__ sum_dyx, const float* __restrict__ gamma,
                                   int c, double* __restrict__ coef /*[4][c]: a, m, mean, k*/) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  double mean, s;
  bn_stats(sum, sumsq, count, eps, ch, mean, s);
  coef[ch] = (gamma ? (double)gamma[ch] : 1.0) * s;
  coef[c + ch] = sum_dy[ch] / count;
  coef[2 * c + ch] = mean;
  coef[3 * c + ch] = s * s * (sum_dyx[ch] - mean * sum_dy[ch]) / count;
}

// per element in float64, one rounding to float32: x - mean needs no float32 rounding of mean on offset channels
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ dy, long long total, int c,
                                                           int hw, const double* __restrict__ coef, float* __restrict__ dx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)((i / hw) % c);
  const double t = (double)dy[i] - coef[c + ch] - ((double)x[i] - coef[2 * c + ch]) * coef[3 * c + ch];
  dx[i] = (float)(coef[ch] * t);
}

// MinibatchLayer pair term, one CTA per kernel k.  Each pair i < j is visited once: c_ij = (g_f[i,k] + g_f[j,k]) e_ijk
// with e_ijk = exp(-Σ_p |A_ikp - A_jkp|), the forward's term bit for bit, goes to the workspace triangle; then
// dA_ikp = -Σ_{j != i} c_ij sgn(A_ikp - A_jkp), j in order, sgn(0) = 0 (Theano's gradient of abs).
__device__ __forceinline__ long long tri_index(int i, int j, int n) { return (long long)i * (2 * n - i - 1) / 2 + (j - i - 1); }

__global__ void __launch_bounds__(256) mb_pair_bwd_kernel(const float* __restrict__ act, const float* __restrict__ g, int n, int d, int K, int P,
                                                          float* __restrict__ pair /*[K][n(n-1)/2]*/, float* __restrict__ dact /*[n][K*P]*/) {
  const int k = blockIdx.x, kp = K * P;
  const long long np = (long long)n * (n - 1) / 2;
  float* ck = pair + (long long)k * np;
  const float* gf = g + d + k;
  for (long long q = threadIdx.x; q < (long long)n * n; q += blockDim.x) {
    const int i = (int)(q / n), j = (int)(q % n);
    if (j <= i) continue;
    float ad = 0.f;
    for (int p = 0; p < P; ++p) ad += fabsf(act[(long long)i * kp + k * P + p] - act[(long long)j * kp + k * P + p]);
    ck[tri_index(i, j, n)] = (gf[(long long)i * (d + K)] + gf[(long long)j * (d + K)]) * expf(-ad);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < n * P; e += blockDim.x) {
    const int i = e / P, p = e % P;
    const float ai = act[(long long)i * kp + k * P + p];
    float s = 0.f;
    for (int j = 0; j < n; ++j) {
      const float df = ai - act[(long long)j * kp + k * P + p];
      if (j == i) continue;
      const float cij = ck[j < i ? tri_index(j, i, n) : tri_index(i, j, n)];
      s += df > 0.f ? cij : (df < 0.f ? -cij : 0.f);
    }
    dact[(long long)i * kp + k * P + p] = -s;
  }
}

// C[m][c] = init[m][c] + Σ_t A(m,t) ks[t] B(t,c), t in order (FFMA, no split): A(m,t) = a[m*sam + t*sat],
// B(t,c) = b[t*sbt + c*sbc]; init and ks nullable.  64 x 64 tiles, 16-deep t steps through shared memory.
__global__ void __launch_bounds__(256) mb_gemm_kernel(const float* __restrict__ a, long long sam, long long sat, const float* __restrict__ b,
                                                      long long sbt, long long sbc, const float* __restrict__ ks, const float* __restrict__ init,
                                                      long long ldi, int M, int N, int T, float* __restrict__ C, long long ldc) {
  __shared__ float As[16][65];
  __shared__ float Bs[16][65];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  float acc[4][4] = {};
  for (int t0 = 0; t0 < T; t0 += 16) {
    for (int e = threadIdx.x; e < 16 * 64; e += 256) {
      const int tt = sat == 1 ? (e & 15) : (e >> 6), mm = sat == 1 ? (e >> 4) : (e & 63);   // the unit stride fastest
      const int t = t0 + tt, m = m0 + mm;
      As[tt][mm] = (t < T && m < M) ? __ldg(a + m * sam + t * sat) * (ks ? __ldg(ks + t) : 1.f) : 0.f;
      const int tb = sbt == 1 ? (e & 15) : (e >> 6), cc = sbt == 1 ? (e >> 4) : (e & 63);
      Bs[tb][cc] = (t0 + tb < T && c0 + cc < N) ? __ldg(b + (t0 + tb) * sbt + (c0 + cc) * sbc) : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int t = 0; t < 16; ++t) {
      float av[4], bv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) { av[r] = As[t][ty + 16 * r]; bv[r] = Bs[t][tx + 16 * r]; }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[r][q] = fmaf(av[r], bv[q], acc[r][q]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int m = m0 + ty + 16 * r, cc = c0 + tx + 16 * q;
      if (m < M && cc < N) C[m * ldc + cc] = (init ? init[m * ldi + cc] : 0.f) + acc[r][q];
    }
}

// through W = theta exp(lws) / r, r = |theta[:, col]|, per column: S = Σ_d theta dW and r² in float64 (block_sum2),
// dtheta = (exp(lws)/r) (dW - theta S / r²), dlws = Σ_d dW W = (exp(lws)/r) S
__global__ void __launch_bounds__(256) mb_param_bwd_kernel(const float* __restrict__ theta, const float* __restrict__ lws,
                                                           const float* __restrict__ dW, int d, int kp, float* __restrict__ dtheta,
                                                           float* __restrict__ dlws) {
  __shared__ double sh[2];
  const int col = blockIdx.x;
  double r2 = 0.0, S = 0.0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    const double t = (double)__ldg(theta + (long long)i * kp + col);
    r2 += t * t;
    S += t * (double)__ldg(dW + (long long)i * kp + col);
  }
  block_sum2(r2, S);
  if (threadIdx.x == 0) { sh[0] = r2; sh[1] = S; }
  __syncthreads();
  r2 = sh[0];
  S = sh[1];
  const double cs = (double)expf(lws[col]) / sqrt(r2);
  if (dlws && threadIdx.x == 0) dlws[col] = (float)(cs * S);
  if (dtheta)
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
      const long long o = (long long)i * kp + col;
      dtheta[o] = (float)(cs * ((double)dW[o] - (double)theta[o] * S / r2));
    }
}

// db[k] = Σ_i g_f[i,k], i in order, float64
__global__ void mb_db_kernel(const float* __restrict__ g, int n, int d, int K, float* __restrict__ db) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += (double)g[(long long)i * (d + K) + d + k];
  db[k] = (float)s;
}

}  // namespace

// workspace: [c][kBnSplits][2] doubles + [3][c] floats -- provided by the caller (ian_api.cu keeps it in the handle)
size_t bn_workspace_bytes(int c) { return (size_t)c * kBnSplits * 2 * sizeof(double) + (size_t)3 * c * sizeof(float); }

// splits per channel of the BatchNorm sums, forward and backward alike
static int bn_splits(int n, int hw) { return hw == 1 ? (n >= 64 ? 8 : 1) : (n < kBnSplits ? n : kBnSplits); }

int launch_bn_batch_stats(const float* x, int n, int c, int hw, double* sum, double* sumsq, void* ws, cudaStream_t st) {
  double* part = reinterpret_cast<double*>(ws);
  const int S = bn_splits(n, hw);
  if (hw == 1)
    bn_partial_dense_kernel<<<dim3((c + 255) / 256, S), 256, 0, st>>>(x, n, c, part);
  else
    bn_partial_kernel<<<dim3(c, S), 256, 0, st>>>(x, n, c, hw, part);
  bn_reduce_kernel<<<(c + 127) / 128, 128, 0, st>>>(part, c, S, sum, sumsq);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_bn_train_normalize(const float* x, int n, int c, int hw, const double* sum, const double* sumsq, double count,
                              const float* gamma, const float* beta, float eps, float alpha, float* running_mean,
                              float* running_inv_std, float* y, void* ws, cudaStream_t st) {
  float* ss = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + (size_t)c * kBnSplits * 2 * sizeof(double));
  bn_finalize_kernel<<<(c + 127) / 128, 128, 0, st>>>(sum, sumsq, count, c, gamma, beta, eps, alpha, running_mean, running_inv_std, ss);
  const long long total = (long long)n * c * hw;
  bn_apply_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, total, c, hw, ss, y);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

size_t mb_workspace_bytes(int n, int K, int P) { return ((size_t)K * P + (size_t)n * K * P) * sizeof(float); }

int launch_minibatch_discrim(const float* x, int n, int d, const float* theta, const float* lws, const float* b, int K, int P,
                             float* out, void* ws, cudaStream_t st) {
  const int kp = K * P;
  float* colscale = reinterpret_cast<float*>(ws);
  float* act = colscale + kp;
  mb_colscale_kernel<<<kp, 256, 0, st>>>(theta, lws, d, kp, colscale);
  mb_activation_kernel<<<dim3((kp + 63) / 64, (n + 15) / 16), 256, 0, st>>>(x, theta, colscale, n, d, kp, act);
  mb_features_kernel<<<n, 128, 0, st>>>(x, act, b, n, d, K, P, out);
  return cudaGetLastError() == cudaSuccess ? 3 : -1;
}

// backward sums: the forward's split structure and bn_reduce_kernel; then this rank's dgamma / dbeta if asked for
int launch_bn_backward_sums(const float* x, const float* dy, int n, int c, int hw, const double* sum, const double* sumsq, double count,
                            float eps, double* sum_dy, double* sum_dyx, float* dgamma, float* dbeta, void* ws, cudaStream_t st) {
  double* part = reinterpret_cast<double*>(ws);
  const int S = bn_splits(n, hw);
  if (hw == 1)
    bn_bwd_partial_dense_kernel<<<dim3((c + 255) / 256, S), 256, 0, st>>>(x, dy, n, c, part);
  else
    bn_bwd_partial_kernel<<<dim3(c, S), 256, 0, st>>>(x, dy, n, c, hw, part);
  bn_reduce_kernel<<<(c + 127) / 128, 128, 0, st>>>(part, c, S, sum_dy, sum_dyx);
  int launches = 2;
  if (dgamma || dbeta) {
    bn_bwd_params_kernel<<<(c + 127) / 128, 128, 0, st>>>(sum, sumsq, count, eps, sum_dy, sum_dyx, c, dgamma, dbeta);
    ++launches;
  }
  return cudaGetLastError() == cudaSuccess ? launches : -1;
}

// the per-channel coefficients ([4][c] doubles) fit in the workspace's partial-sum area
int launch_bn_backward_dx(const float* x, const float* dy, int n, int c, int hw, const double* sum, const double* sumsq, double count,
                          const double* sum_dy, const double* sum_dyx, const float* gamma, float eps, float* dx, void* ws, cudaStream_t st) {
  double* coef = reinterpret_cast<double*>(ws);
  bn_bwd_coef_kernel<<<(c + 127) / 128, 128, 0, st>>>(sum, sumsq, count, eps, sum_dy, sum_dyx, gamma, c, coef);
  const long long total = (long long)n * c * hw;
  bn_bwd_apply_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, dy, total, c, hw, coef, dx);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

// workspace: colscale [kp] | act [n][kp] | dact [n][kp] | pair triangles [K][n(n-1)/2] | dW [d][kp], floats
size_t mb_bwd_workspace_bytes(int n, int d, int K, int P) {
  const size_t kp = (size_t)K * P;
  return (kp + 2 * (size_t)n * kp + (size_t)K * ((size_t)n * (n - 1) / 2) + (size_t)d * kp) * sizeof(float);
}

int launch_minibatch_discrim_bwd(const float* x, int n, int d, const float* theta, const float* lws, int K, int P, const float* g,
                                 float* dx, float* dtheta, float* dlws, float* db, void* ws, cudaStream_t st) {
  const int kp = K * P;
  float* colscale = reinterpret_cast<float*>(ws);
  float* act = colscale + kp;
  float* dact = act + (size_t)n * kp;
  float* pair = dact + (size_t)n * kp;
  float* dW = pair + (size_t)K * ((size_t)n * (n - 1) / 2);
  int launches = 0;
  if (dx || dtheta || dlws) {
    mb_colscale_kernel<<<kp, 256, 0, st>>>(theta, lws, d, kp, colscale);
    mb_activation_kernel<<<dim3((kp + 63) / 64, (n + 15) / 16), 256, 0, st>>>(x, theta, colscale, n, d, kp, act);
    mb_pair_bwd_kernel<<<K, 256, 0, st>>>(act, g, n, d, K, P, pair, dact);
    launches += 3;
  }
  if (dx) {                                   // dx = g_x + (dA colscale) theta^T
    mb_gemm_kernel<<<dim3((d + 63) / 64, (n + 63) / 64), 256, 0, st>>>(dact, kp, 1, theta, 1, kp, colscale, g, d + K, n, d, kp, dx, d);
    ++launches;
  }
  if (dtheta || dlws) {                       // dW = x^T dA, then the column-norm chain
    mb_gemm_kernel<<<dim3((kp + 63) / 64, (d + 63) / 64), 256, 0, st>>>(x, 1, d, dact, kp, 1, nullptr, nullptr, 0, d, kp, n, dW, kp);
    mb_param_bwd_kernel<<<kp, 256, 0, st>>>(theta, lws, dW, d, kp, dtheta, dlws);
    launches += 2;
  }
  if (db) {
    mb_db_kernel<<<(K + 127) / 128, 128, 0, st>>>(g, n, d, K, db);
    ++launches;
  }
  return cudaGetLastError() == cudaSuccess ? launches : -1;
}

}  // namespace ian
