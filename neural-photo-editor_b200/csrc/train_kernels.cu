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

}  // namespace

// workspace: [c][kBnSplits][2] doubles + [3][c] floats -- provided by the caller (ian_api.cu keeps it in the handle)
size_t bn_workspace_bytes(int c) { return (size_t)c * kBnSplits * 2 * sizeof(double) + (size_t)3 * c * sizeof(float); }

int launch_bn_batch_stats(const float* x, int n, int c, int hw, double* sum, double* sumsq, void* ws, cudaStream_t st) {
  double* part = reinterpret_cast<double*>(ws);
  int S;
  if (hw == 1) {
    S = n >= 64 ? 8 : 1;
    bn_partial_dense_kernel<<<dim3((c + 255) / 256, S), 256, 0, st>>>(x, n, c, part);
  } else {
    S = n < kBnSplits ? n : kBnSplits;
    bn_partial_kernel<<<dim3(c, S), 256, 0, st>>>(x, n, c, hw, part);
  }
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

}  // namespace ian
