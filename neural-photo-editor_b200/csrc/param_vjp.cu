// param_vjp.cu -- the small reductions of the IAN_simple decoder's parameter VJP (ian_decode_param_vjp_*): dec_out's
// weight gradient and the BatchNorm beta / gamma gradients.  Both are two-level and fixed-order (per-chunk partial sums in
// a fixed lane order, then the chunks added in chunk order), so a repeated call is bit-identical; no atomics.
#include "edge.h"
#include "tapgemm.h"

namespace ian {

namespace {

// dec_out (layers.py:436-483 with W (128, 3, 5, 5)): y[co][2p+r][2q+s] = sum_{ci,d,e} h3[ci][p+d][q+e] W[ci][co][2+2d-r][2+2e-s]
// so for tap (ki, kj): r = ki & 1, d = (ki - 2 + r) / 2 (same for kj) and
//   dW[ci][co][ki][kj] = sum_{n,p,q} seed[n][co][2p+r][2q+s] * h3[n][p+d][q+e][ci],   seed = dx_hat * (1 - x_hat^2).
// Block (tap, 32-channel group, pixel chunk); lane = channel, warp = one of 8 interleaved pixel streams.
__global__ void __launch_bounds__(256) decout_wgrad_kernel(const float* __restrict__ seed, const __nv_bfloat16* __restrict__ h3,
                                                           long long plane, int n, float* __restrict__ part) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  __shared__ float red[8][32][3];
  const int t = blockIdx.x, ci = blockIdx.y * 32 + (threadIdx.x & 31), lane8 = threadIdx.x >> 5;
  const int ki = t / 5, kj = t % 5;
  const int r = ki & 1, s = kj & 1, d = (ki - 2 + r) / 2, e = (kj - 2 + s) / 2;
  const long long K = (long long)n * 1024;
  const long long k0 = K * blockIdx.z / gridDim.z, k1 = K * (blockIdx.z + 1) / gridDim.z;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (long long m = k0 + lane8; m < k1; m += 8) {
    const int img = (int)(m >> 10), p = (int)(m >> 5) & 31, q = (int)m & 31;
    const int pp = p + d, qq = q + e;
    if (pp < 0 || pp >= 32 || qq < 0 || qq >= 32) continue;
    const long long ai = ((long long)(img * 32 + pp) * 32 + qq) * 128 + ci;
    const float av = __bfloat162float(h3[ai]) + __bfloat162float(h3[ai + plane]);
    const float* sp = seed + (long long)img * 3 * 4096 + (2 * p + r) * 64 + 2 * q + s;
    a0 = fmaf(__ldg(sp), av, a0);
    a1 = fmaf(__ldg(sp + 4096), av, a1);
    a2 = fmaf(__ldg(sp + 8192), av, a2);
  }
  red[lane8][threadIdx.x & 31][0] = a0;
  red[lane8][threadIdx.x & 31][1] = a1;
  red[lane8][threadIdx.x & 31][2] = a2;
  __syncthreads();
  if (threadIdx.x < 96) {
    const int c = threadIdx.x / 3, co = threadIdx.x % 3;
    float v = red[0][c][co];
    for (int l = 1; l < 8; ++l) v += red[l][c][co];
    part[((long long)blockIdx.z * 25 + t) * 384 + (blockIdx.y * 32 + c) * 3 + co] = v;
  }
}

// part [chunk][25][128][3] -> dW (128, 3, 5, 5), chunks added in order
__global__ void decout_wgrad_finalize_kernel(const float* __restrict__ part, int nchunk, float* __restrict__ out, int accumulate) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 25 * 384) return;
  const int t = i / 384, ci = (i % 384) / 3, co = i % 3;
  float v = part[i];
  for (int k = 1; k < nchunk; ++k) v += part[(long long)k * 25 * 384 + i];
  const int dst = (ci * 3 + co) * 25 + t;
  out[dst] = accumulate ? out[dst] + v : v;
}

// Inference BatchNorm y = (x - mean) * inv_std * gamma + beta, h = rectify(y), with dL/dh given:
//   dL/dy = dL/dh * (h > 0);  d beta_c = sum dL/dy;  d gamma_c = sum dL/dy * (x - mean_c) * inv_std_c.
// Elements (row, c) at row * C + c; the sums run over rows.  fc2 = 1: bnorm_dec_fc2 is per feature of the NHWC-ordered
// column c = hw*1024 + ch, whose reference index is j = ch*16 + hw.  Block (32 channels, row chunk), 8 row streams.
__global__ void __launch_bounds__(256) bn_param_bwd_kernel(const __nv_bfloat16* __restrict__ dh, long long dh_plane,
                                                           const __nv_bfloat16* __restrict__ h,
                                                           const __nv_bfloat16* __restrict__ x, long long x_plane,
                                                           const float* __restrict__ mean, const float* __restrict__ istd,
                                                           int C, long long R, int fc2, float* __restrict__ part) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  __shared__ float red[8][32][2];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), lane8 = threadIdx.x >> 5;
  const int j = fc2 ? (c % 1024) * 16 + c / 1024 : c;
  const float mu = __ldg(mean + j), is = __ldg(istd + j);
  const long long r0 = R * blockIdx.y / gridDim.y, r1 = R * (blockIdx.y + 1) / gridDim.y;
  float sb = 0.f, sg = 0.f;
  for (long long r = r0 + lane8; r < r1; r += 8) {
    const long long i = r * C + c;
    if (!(__bfloat162float(h[i]) > 0.f)) continue;
    const float dy = __bfloat162float(dh[i]) + __bfloat162float(dh[i + dh_plane]);
    const float xn = (__bfloat162float(x[i]) + __bfloat162float(x[i + x_plane]) - mu) * is;
    sb += dy;
    sg = fmaf(dy, xn, sg);
  }
  red[lane8][threadIdx.x & 31][0] = sb;
  red[lane8][threadIdx.x & 31][1] = sg;
  __syncthreads();
  if (threadIdx.x < 64) {
    const int cc = threadIdx.x >> 1, which = threadIdx.x & 1;
    float v = red[0][cc][which];
    for (int l = 1; l < 8; ++l) v += red[l][cc][which];
    part[((long long)blockIdx.y * 2 + which) * C + blockIdx.x * 32 + cc] = v;
  }
}

__global__ void bn_param_finalize_kernel(const float* __restrict__ part, int nchunk, int C, int fc2, float* __restrict__ dbeta,
                                         float* __restrict__ dgamma, int accumulate) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * C) return;
  const int which = i / C, c = i % C;
  float* out = which ? dgamma : dbeta;
  if (!out) return;
  float v = part[i];
  for (int k = 1; k < nchunk; ++k) v += part[(long long)k * 2 * C + i];
  const int j = fc2 ? (c % 1024) * 16 + c / 1024 : c;
  out[j] = accumulate ? out[j] + v : v;
}

}  // namespace

int decout_wgrad_chunks(int n) { return n < 16 ? n : 16; }
int bn_param_chunks(int C, long long R) {
  long long k = R / 512;                                // >= 512 rows per chunk
  const long long want = (2LL * tc_num_sms() + C / 32 - 1) / (C / 32);   // about two waves of blocks
  if (k > want) k = want;
  if (k > 64) k = 64;
  return k < 1 ? 1 : (int)k;
}

int launch_decout_wgrad(const float* seed, const __nv_bfloat16* h3, long long plane, int n, float* part, float* out,
                        int accumulate, cudaStream_t st) {
  const int nc = decout_wgrad_chunks(n);
  if (launch_pdl(decout_wgrad_kernel, dim3(25, 4, nc), dim3(256), 0, st, seed, h3, plane, n, part) != cudaSuccess) return -1;
  if (launch_pdl(decout_wgrad_finalize_kernel, dim3((25 * 384 + 255) / 256), dim3(256), 0, st, (const float*)part, nc, out,
                 accumulate) != cudaSuccess)
    return -1;
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_bn_param_bwd(const __nv_bfloat16* dh, long long dh_plane, const __nv_bfloat16* h, const __nv_bfloat16* x,
                        long long x_plane, const float* mean, const float* istd, int C, long long R, int fc2, float* part,
                        float* dbeta, float* dgamma, int accumulate, cudaStream_t st) {
  const int nc = bn_param_chunks(C, R);
  if (launch_pdl(bn_param_bwd_kernel, dim3(C / 32, nc), dim3(256), 0, st, dh, dh_plane, h, x, x_plane, mean, istd, C, R, fc2,
                 part) != cudaSuccess)
    return -1;
  if (launch_pdl(bn_param_finalize_kernel, dim3((2 * C + 255) / 256), dim3(256), 0, st, (const float*)part, nc, C, fc2, dbeta,
                 dgamma, accumulate) != cudaSuccess)
    return -1;
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

}  // namespace ian
