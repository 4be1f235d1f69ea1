// disc_kernels.cu -- the IAN's discriminator head l_discrim under deterministic=True (ian_discriminate_*,
// ian_discriminate_vjp_*; DESIGN section 5.6n).  The trunk is the encoder to enc_conv4 (a4, split planes NHWC); the
// MinibatchLayer between the two kernels of each direction is train_kernels.cu's.
//   disc_pool       : GlobalPoolLayer, the mean of a4 over its 4 x 4 pixels -> (n,1024) float32, pixels added in order
//   disc_head       : the dense layer 1524 -> U without bias and its nonlinearity: logits = [pool | f] W, p = sigmoid (U = 1)
//                     or softmax with its max subtracted (U = 3).  One CTA per sample, FFMA, a fixed summation order
//   disc_head_bwd   : its adjoint d[pool | f] = dlogits W^T, U products per element in u order
//   disc_cotangent  : d pool -> the cotangent of a4, c4 = broadcast(d pool / 16) (n,1024,4,4) float32 NCHW
// A feature value is what the encoder stores: hi + lo of the split planes, or hi alone in bf16 mode (launch_feat_store's rule).
//
// The batch-statistics BatchNorm stacks (ian_api.cu's BnStack; DESIGN section 5.6o) -- the training-mode trunk
// (ian_discriminate_train*: bnorm2..4 on enc_conv2..4) and the IAN_simple decoder in training mode (ian_decode_train*;
// DESIGN section 5.6p: bnorm_dec_fc2 with hw = 1 and c = its 16384 library columns, bnorm_dc1..3) -- share these kernels on
// the layers' raw sums in whole-call float32 NHWC buffers (n, HW, C), channel c of pixel p of image i at (i HW + p) C + c:
//   nhwc_bn_partial  : per image and channel, Σu and Σu·v in float64 over the image's pixels in order (u = v = x: the
//                      forward's Σx, Σx²; u = dy, v = x: the backward's Σdy, Σdy·x)
//   nhwc_bn_stats    : the images' partials added in image order, so the sums do not depend on the chunking; mean and
//                      inv_std = 1/sqrt(var + eps) as bn_finalize_kernel forms them (biased var), float32 copies for the callers
//   nhwc_bn_act      : y = (x - mean) (gamma inv_std) + beta, a = fmaf(act_abs, |y|, act_lin y) -> split planes (hi only in
//                      bf16 mode): LeakyReLU(0.2) with 0.4, 0.6 (the trunk), rectify with 0.5, 0.5 (the decoder)
//   nhwc_bn_coef     : bn_bwd_coef_kernel's coefficients (train_kernels.cu) from the whole-call sums, in its own rounding
//   nhwc_bn_dx       : dx per element in float64, rounded once as bn_bwd_apply_kernel does -> split planes
// Each stack's own kernels:
//   disc_train_cot   : the pool's adjoint times lrelu'(y4): dy4 = d pool / 16 * (y4 > 0 ? 1 : 0.2), float32
//   dec_train_dy     : dy = dL/dh (hi + lo of split planes) * (y > 0), float32: bnorm_dc3's cotangent from the seed kernel
//   dec_bn_grads     : d beta = Σdy, d gamma = inv_std (Σdy·x - mean Σdy) in float64 from the whole-call sums, written in
//                      the reference's feature order
//   dec_stats_out    : the statistics in the reference's feature order
// bnorm_dec_fc2's library column c = hw 1024 + ch is the reference's feature ch 16 + hw.
#include "edge.h"

namespace ian {

namespace {

constexpr int kC4 = 1024, kPool = 16, kIn = kC4 + kDiscKernels, kHeadThreads = 128;

// thread (k, c): coalesced over channels
__global__ void __launch_bounds__(256) disc_pool_kernel(const __nv_bfloat16* __restrict__ a4, long long plane, int passes, int n,
                                                        float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (o >= (long long)n * kC4) return;
  const long long k = o / kC4, c = o % kC4;
  float s = 0.f;
#pragma unroll
  for (int p = 0; p < kPool; ++p) {
    const long long i = (k * kPool + p) * kC4 + c;
    const float hi = __bfloat162float(a4[i]);
    s += passes == 1 ? hi : hi + __bfloat162float(a4[plane + i]);
  }
  out[o] = s * (1.f / kPool);                            // T.mean: the sum over 16, exact as a power of two
}

// thread t sums inputs t, t + 128, ... in order; the warps' sums meet by a fixed butterfly, then warp 0..3 in order
__global__ void __launch_bounds__(kHeadThreads) disc_head_kernel(const float* __restrict__ in, const float* __restrict__ W, int U,
                                                                 float* __restrict__ logits, float* __restrict__ p) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[kHeadThreads / 32][kDiscMaxUnits];
  const int i = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float* row = in + (long long)i * kIn;
  float acc[kDiscMaxUnits] = {0.f, 0.f, 0.f};
  for (int j = t; j < kIn; j += kHeadThreads) {
    const float v = row[j];
#pragma unroll
    for (int u = 0; u < kDiscMaxUnits; ++u)
      if (u < U) acc[u] = fmaf(v, W[j * U + u], acc[u]);
  }
#pragma unroll
  for (int u = 0; u < kDiscMaxUnits; ++u) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[u] += __shfl_xor_sync(0xffffffffu, acc[u], o);
    if (lane == 0) red[warp][u] = acc[u];
  }
  __syncthreads();
  if (t != 0) return;
  float l[kDiscMaxUnits];
  for (int u = 0; u < U; ++u) {
    float s = red[0][u];
    for (int w = 1; w < kHeadThreads / 32; ++w) s += red[w][u];
    l[u] = s;
    logits[i * U + u] = s;
  }
  if (!p) return;
  if (U == 1) {
    p[i] = 1.f / (1.f + expf(-l[0]));
    return;
  }
  float m = l[0];
  for (int u = 1; u < U; ++u) m = fmaxf(m, l[u]);
  float e[kDiscMaxUnits], s = 0.f;
  for (int u = 0; u < U; ++u) {
    e[u] = expf(l[u] - m);
    s += e[u];
  }
  for (int u = 0; u < U; ++u) p[i * U + u] = e[u] / s;
}

__global__ void __launch_bounds__(256) disc_head_bwd_kernel(const float* __restrict__ dl, const float* __restrict__ W, int U, int n,
                                                            float* __restrict__ g) {
  pdl_trigger();
  pdl_wait();
  const long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (o >= (long long)n * kIn) return;
  const long long i = o / kIn, j = o % kIn;
  float s = 0.f;
  for (int u = 0; u < U; ++u) s = fmaf(dl[i * U + u], W[j * U + u], s);
  g[o] = s;
}

__global__ void __launch_bounds__(256) disc_cotangent_kernel(const float* __restrict__ dpool, int n, float* __restrict__ c4) {
  pdl_trigger();
  pdl_wait();
  const long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (o >= (long long)n * kC4 * kPool) return;
  c4[o] = dpool[o / kPool] * (1.f / kPool);
}

unsigned blocks_of(long long total) { return (unsigned)((total + 255) / 256); }

// thread (image, channel): coalesced over channels, the image's pixels in order
__global__ void __launch_bounds__(128) nhwc_bn_partial_kernel(const float* __restrict__ u, const float* __restrict__ v, int hw, int c,
                                                              double* __restrict__ part /*[n][2][c]*/) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (ch >= c) return;
  const long long base = (long long)i * hw * c + ch;
  double s = 0.0, q = 0.0;                               // float64 from the first term: a product of two float32 is exact
  for (int p = 0; p < hw; ++p) {
    const double a = (double)__ldg(u + base + (long long)p * c);
    s += a;
    q += a * (double)__ldg(v + base + (long long)p * c);
  }
  part[((long long)i * 2) * c + ch] = s;
  part[((long long)i * 2 + 1) * c + ch] = q;
}

// sums[2][c] = the partials of images 0..n-1 in order; with count > 0 also mean_f / inv_std_f (the forward's statistics)
__global__ void nhwc_bn_stats_kernel(const double* __restrict__ part, int n, int c, double count, float eps, double* __restrict__ sums,
                                     float* __restrict__ mean_f, float* __restrict__ inv_std_f) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  double s = 0.0, q = 0.0;
  for (int i = 0; i < n; ++i) {
    s += part[((long long)i * 2) * c + ch];
    q += part[((long long)i * 2 + 1) * c + ch];
  }
  sums[ch] = s;
  sums[c + ch] = q;
  if (!mean_f) return;
  const double mean = s / count;
  double var = q / count - mean * mean;                  // biased variance, as theano's x.var(axes)
  if (var < 0.0) var = 0.0;
  mean_f[ch] = (float)mean;
  inv_std_f[ch] = (float)(1.0 / sqrt(var + (double)eps));
}

// lasagne's order: (x - mean) * (gamma * inv_std) + beta
__device__ __forceinline__ float bn_train_y(float x, int ch, const float* mean, const float* inv_std, const float* gamma,
                                            const float* beta) {
  return (x - __ldg(mean + ch)) * (__ldg(gamma + ch) * __ldg(inv_std + ch)) + __ldg(beta + ch);
}

// act_abs, act_lin: the activation as the tap-GEMM epilogue forms it
__global__ void __launch_bounds__(256) nhwc_bn_act_kernel(const float* __restrict__ x, long long total, int c, const float* __restrict__ mean,
                                                          const float* __restrict__ inv_std, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float act_abs, float act_lin, int passes,
                                                          __nv_bfloat16* __restrict__ out, long long plane) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float y = bn_train_y(x[i], (int)(i % c), mean, inv_std, gamma, beta);
  const float a = fmaf(act_abs, fabsf(y), act_lin * y);
  __nv_bfloat16 hi, lo;
  split_bf16(a, hi, lo);
  out[i] = hi;
  if (passes != 1) out[plane + i] = lo;
}

__global__ void __launch_bounds__(256) disc_train_cot_kernel(const float* __restrict__ dpool, const float* __restrict__ x4, int n,
                                                             const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float* __restrict__ dy) {
  const long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (o >= (long long)n * kPool * kC4) return;
  const int ch = (int)(o % kC4);
  const float y = bn_train_y(x4[o], ch, mean, inv_std, gamma, beta);
  dy[o] = dpool[(o / (kPool * kC4)) * kC4 + ch] * (1.f / kPool) * (y > 0.f ? 1.f : 0.2f);
}

// dx = a (dy - m - (x - mean) k), a = gamma s, m = Σdy/N, k = s² (Σdy·x - mean Σdy)/N, s = inv_std in float64: the coefficients
// of bn_bwd_coef_kernel (train_kernels.cu), kept apart because the two compile differently: here Σx²/N - mean² is one fused
// multiply-add, there (bn_stats) mean² is rounded before the subtraction, so s can differ in its last bit
__global__ void nhwc_bn_coef_kernel(const double* __restrict__ fsum, const double* __restrict__ bsum, double count, float eps,
                                    const float* __restrict__ gamma, int c, double* __restrict__ coef /*[4][c]*/) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  const double mean = fsum[ch] / count;
  double var = fsum[c + ch] / count - mean * mean;
  if (var < 0.0) var = 0.0;
  const double s = 1.0 / sqrt(var + (double)eps);
  coef[ch] = (double)gamma[ch] * s;
  coef[c + ch] = bsum[ch] / count;
  coef[2 * c + ch] = mean;
  coef[3 * c + ch] = s * s * (bsum[c + ch] - mean * bsum[ch]) / count;
}

__global__ void __launch_bounds__(256) nhwc_bn_dx_kernel(const float* __restrict__ x, const float* __restrict__ dy, long long total, int c,
                                                         const double* __restrict__ coef, int passes, __nv_bfloat16* __restrict__ out,
                                                         long long plane) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)(i % c);
  const double t = (double)dy[i] - coef[c + ch] - ((double)x[i] - coef[2 * c + ch]) * coef[3 * c + ch];
  __nv_bfloat16 hi, lo;
  split_bf16((float)(coef[ch] * t), hi, lo);
  out[i] = hi;
  if (passes != 1) out[plane + i] = lo;
}

__global__ void __launch_bounds__(256) dec_train_dy_kernel(const __nv_bfloat16* __restrict__ dh, long long plane,
                                                           const float* __restrict__ x, long long total, int c,
                                                           const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           float* __restrict__ dy) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float y = bn_train_y(x[i], (int)(i % c), mean, inv_std, gamma, beta);
  dy[i] = y > 0.f ? __bfloat162float(dh[i]) + __bfloat162float(dh[plane + i]) : 0.f;
}

__device__ __forceinline__ int ref_feature(int col, int fc2) { return fc2 ? (col % 1024) * 16 + col / 1024 : col; }

__global__ void dec_bn_grads_kernel(const double* __restrict__ fsum, const double* __restrict__ bsum, double count, float eps,
                                    int c, int fc2, float* __restrict__ dbeta, float* __restrict__ dgamma) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  const int j = ref_feature(ch, fc2);
  if (dbeta) dbeta[j] = (float)bsum[ch];
  if (!dgamma) return;
  const double mean = fsum[ch] / count;
  double var = fsum[c + ch] / count - mean * mean;
  if (var < 0.0) var = 0.0;
  dgamma[j] = (float)((bsum[c + ch] - mean * bsum[ch]) / sqrt(var + (double)eps));
}

// in, out: [2][total] (mean | inv_std); the first fc2_cols columns are bnorm_dec_fc2's
__global__ void dec_stats_out_kernel(const float* __restrict__ in, int total, int fc2_cols, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * total) return;
  const int r = i / total, col = i % total;
  out[r * total + (col < fc2_cols ? ref_feature(col, 1) : col)] = in[i];
}

}  // namespace

int launch_disc_pool(const __nv_bfloat16* a4, long long plane, int passes, int n, float* out, cudaStream_t st) {
  return launch_pdl(disc_pool_kernel, dim3(blocks_of((long long)n * kC4)), dim3(256), 0, st, a4, plane, passes, n, out) ==
                 cudaSuccess ? 1 : -1;
}

int launch_disc_head(const float* in, const float* W, int U, int n, float* logits, float* p, cudaStream_t st) {
  if (U < 1 || U > kDiscMaxUnits) return -1;
  return launch_pdl(disc_head_kernel, dim3(n), dim3(kHeadThreads), 0, st, in, W, U, logits, p) == cudaSuccess ? 1 : -1;
}

int launch_disc_head_bwd(const float* dlogits, const float* W, int U, int n, float* g, cudaStream_t st) {
  return launch_pdl(disc_head_bwd_kernel, dim3(blocks_of((long long)n * kIn)), dim3(256), 0, st, dlogits, W, U, n, g) ==
                 cudaSuccess ? 1 : -1;
}

int launch_disc_cotangent(const float* dpool, int n, float* c4, cudaStream_t st) {
  return launch_pdl(disc_cotangent_kernel, dim3(blocks_of((long long)n * kC4 * kPool)), dim3(256), 0, st, dpool, n, c4) ==
                 cudaSuccess ? 1 : -1;
}

int launch_nhwc_bn_sums(const float* u, const float* v, int n, int hw, int c, double count, float eps, double* part, double* sums,
                        float* mean_f, float* inv_std_f, cudaStream_t st) {
  nhwc_bn_partial_kernel<<<dim3((c + 127) / 128, n), 128, 0, st>>>(u, v, hw, c, part);
  nhwc_bn_stats_kernel<<<(c + 127) / 128, 128, 0, st>>>(part, n, c, count, eps, sums, mean_f, inv_std_f);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_nhwc_bn_act(const float* x, long long total, int c, const float* mean, const float* inv_std, const float* gamma,
                       const float* beta, float act_abs, float act_lin, int passes, __nv_bfloat16* out, long long plane,
                       cudaStream_t st) {
  nhwc_bn_act_kernel<<<blocks_of(total), 256, 0, st>>>(x, total, c, mean, inv_std, gamma, beta, act_abs, act_lin, passes, out, plane);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_disc_train_cotangent(const float* dpool, const float* x4, int n, const float* mean, const float* inv_std,
                                const float* gamma, const float* beta, float* dy, cudaStream_t st) {
  disc_train_cot_kernel<<<blocks_of((long long)n * kPool * kC4), 256, 0, st>>>(dpool, x4, n, mean, inv_std, gamma, beta, dy);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_nhwc_bn_coef(const double* fsum, const double* bsum, double count, float eps, const float* gamma, int c, double* coef,
                        cudaStream_t st) {
  nhwc_bn_coef_kernel<<<(c + 127) / 128, 128, 0, st>>>(fsum, bsum, count, eps, gamma, c, coef);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_nhwc_bn_dx(const float* x, const float* dy, long long total, int c, const double* coef, int passes, __nv_bfloat16* out,
                      long long plane, cudaStream_t st) {
  nhwc_bn_dx_kernel<<<blocks_of(total), 256, 0, st>>>(x, dy, total, c, coef, passes, out, plane);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_dec_train_dy(const __nv_bfloat16* dh, long long plane, const float* x, long long total, int c, const float* mean,
                        const float* inv_std, const float* gamma, const float* beta, float* dy, cudaStream_t st) {
  dec_train_dy_kernel<<<blocks_of(total), 256, 0, st>>>(dh, plane, x, total, c, mean, inv_std, gamma, beta, dy);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_dec_bn_grads(const double* fsum, const double* bsum, double count, float eps, int c, int fc2, float* dbeta,
                        float* dgamma, cudaStream_t st) {
  dec_bn_grads_kernel<<<(c + 127) / 128, 128, 0, st>>>(fsum, bsum, count, eps, c, fc2, dbeta, dgamma);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_dec_stats_out(const float* in, int total, int fc2_cols, float* out, cudaStream_t st) {
  dec_stats_out_kernel<<<blocks_of(2LL * total), 256, 0, st>>>(in, total, fc2_cols, out);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ian
