// disc_kernels.cu -- the IAN's discriminator head l_discrim under deterministic=True (ian_discriminate_*,
// ian_discriminate_vjp_*; DESIGN section 5.6n).  The trunk is the encoder to enc_conv4 (a4, split planes NHWC); the
// MinibatchLayer between the two kernels of each direction is train_kernels.cu's.
//   disc_pool       : GlobalPoolLayer, the mean of a4 over its 4 x 4 pixels -> (n,1024) float32, pixels added in order
//   disc_head       : the dense layer 1524 -> U without bias and its nonlinearity: logits = [pool | f] W, p = sigmoid (U = 1)
//                     or softmax with its max subtracted (U = 3).  One CTA per sample, FFMA, a fixed summation order
//   disc_head_bwd   : its adjoint d[pool | f] = dlogits W^T, U products per element in u order
//   disc_cotangent  : d pool -> the cotangent of a4, c4 = broadcast(d pool / 16) (n,1024,4,4) float32 NCHW
// A feature value is what the encoder stores: hi + lo of the split planes, or hi alone in bf16 mode (launch_feat_store's rule).
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

}  // namespace ian
