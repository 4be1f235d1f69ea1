// enc_vjp.cu -- the small kernels of the encoder vector-Jacobian product dx = (dz/dx)^T dz (ian_encode_vjp_*).
// The heavy layers of that chain are tap-GEMMs (tapgemm.h) on weight tiles permuted from the forward ones; what is left:
//   made_iaf_bwd : backward of the MADE/IAF latent flow (IAN.py:126-128 / IANv1.py:121-123), one block per sample
//   seed         : dz_iaf -> gradient of the encoder head's pre-BatchNorm GEMM output (mu | logsigma columns)
//   fc1_bwd      : float32 gradient of enc_fc1's output -> ReLU / ELU derivative * bnorm_enc_fc1 scale, split planes
//   permute      : forward weight tiles [t][R][C] -> backward tiles [t'][C][R] (t' = t or 24 - t), both bf16 planes
// and the two of the encoder Jacobian-vector product dz = (dz/dx) v (ian_encode_jvp_*) after its tangent tap-GEMMs:
//   sample_tangent   : tangent of the encoder head [t_mu | t_ls] -> tangent of z_iaf = mu (+ exp(logsigma) eps)
//   made_iaf_tangent : forward mode through the MADE/IAF latent flow, one block per sample
#include "edge.h"

namespace ian {

namespace {

// Forward (made_iaf_kernel, edge_kernels.cu), per net in {mu, ls}:
//   pu = z0 W0 + b0, u = rect(pu);  ph = u W0 + b0, h = rect(ph);  o = b1 + bd + h W1 + u Wd
//   z  = (z0 - o_mu) / exp(o_ls)
// Backward: g_mu = -dz / exp(o_ls), g_ls = -dz * z, dz0 = dz / exp(o_ls), then per net
//   dh = W1 g;  du = Wd g + W0 (dh * rect'(ph));  dz0 += W0 (du * rect'(pu))
// rect = lasagne rectify 0.5 (x + |x|), whose Theano derivative is 0.5 (1 + sgn x): 1, 0 and 1/2 at exactly 0.
// The forward sums are recomputed in made_iaf_kernel's fmaf order, so o, z and the masks are its values.
__device__ __forceinline__ float rect_grad(float a) { return a > 0.f ? 1.f : (a < 0.f ? 0.f : 0.5f); }

__global__ void __launch_bounds__(128) made_iaf_bwd_kernel(const float* __restrict__ z0, const float* __restrict__ mw,
                                                           const float* __restrict__ mb, const float* __restrict__ dz,
                                                           float* __restrict__ dzi, int n) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  __shared__ float zs[100];
  __shared__ float us[2][100], pus[2][100], phs[2][100], hs[2][100];
  __shared__ float gs[2][100], dphs[2][100], dpus[2][100];
  const int k = blockIdx.x, j = threadIdx.x;
  if (j < 100) zs[j] = z0[k * 100 + j];
  __syncthreads();
  if (j < 100) {
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W0 = mw + (net * 3 + 0) * 10000;
      float a = mb[(net * 3 + 0) * 100 + j];
      for (int i = 0; i < 100; ++i) a = fmaf(zs[i], W0[i * 100 + j], a);
      pus[net][j] = a;
      us[net][j] = 0.5f * (a + fabsf(a));
    }
  }
  __syncthreads();
  if (j < 100) {
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W0 = mw + (net * 3 + 0) * 10000;
      float a = mb[(net * 3 + 0) * 100 + j];
      for (int i = 0; i < 100; ++i) a = fmaf(us[net][i], W0[i * 100 + j], a);
      phs[net][j] = a;
      hs[net][j] = 0.5f * (a + fabsf(a));
    }
  }
  __syncthreads();
  float dzj = 0.f;
  if (j < 100) {
    float o[2];
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W1 = mw + (net * 3 + 1) * 10000;
      const float* Wd = mw + (net * 3 + 2) * 10000;
      float a = mb[(net * 3 + 1) * 100 + j] + mb[(net * 3 + 2) * 100 + j];
      float a1 = 0.f, a2 = 0.f;
      for (int i = 0; i < 100; ++i) {
        a1 = fmaf(hs[net][i], W1[i * 100 + j], a1);
        a2 = fmaf(us[net][i], Wd[i * 100 + j], a2);
      }
      o[net] = a + a1 + a2;
    }
    const float e = expf(o[1]);
    const float z = (zs[j] - o[0]) / e;
    const float d = dz[k * 100 + j];
    dzj = d / e;
    gs[0][j] = -dzj;
    gs[1][j] = -d * z;
  }
  __syncthreads();
  // dh = W1 g and the direct part of du = Wd g (row j of each matrix: unit j's fan-out)
  float du[2] = {0.f, 0.f};
  if (j < 100) {
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W1 = mw + (net * 3 + 1) * 10000 + j * 100;
      const float* Wd = mw + (net * 3 + 2) * 10000 + j * 100;
      float dh = 0.f, dd = 0.f;
      for (int i = 0; i < 100; ++i) {
        dh = fmaf(W1[i], gs[net][i], dh);
        dd = fmaf(Wd[i], gs[net][i], dd);
      }
      dphs[net][j] = dh * rect_grad(phs[net][j]);
      du[net] = dd;
    }
  }
  __syncthreads();
  if (j < 100) {
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W0 = mw + (net * 3 + 0) * 10000 + j * 100;
      float a = du[net];
      for (int i = 0; i < 100; ++i) a = fmaf(W0[i], dphs[net][i], a);
      dpus[net][j] = a * rect_grad(pus[net][j]);
    }
  }
  __syncthreads();
  if (j < 100) {
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W0 = mw + (net * 3 + 0) * 10000 + j * 100;
      for (int i = 0; i < 100; ++i) dzj = fmaf(W0[i], dpus[net][i], dzj);
    }
    dzi[k * 100 + j] = dzj;
  }
}

// Forward mode of the same flow: with the forward recomputed as above (made_iaf_kernel's fmaf order),
//   t_u = rect'(pu) (t_z0 W0);  t_h = rect'(ph) (t_u W0);  t_o = t_h W1 + t_u Wd   per net
//   t_z = (t_z0 - t_o_mu) / exp(o_ls) - z t_o_ls
// with the backward's rect' (1/2 at exactly 0), so this is the exact transpose of made_iaf_bwd_kernel's linear map.
__global__ void __launch_bounds__(128) made_iaf_tangent_kernel(const float* __restrict__ z0, const float* __restrict__ tz0,
                                                               const float* __restrict__ mw, const float* __restrict__ mb,
                                                               float* __restrict__ tz, int n) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  __shared__ float zs[100], tzs[100];
  __shared__ float us[2][100], hs[2][100], tus[2][100], ths[2][100];
  const int k = blockIdx.x, j = threadIdx.x;
  if (j < 100) {
    zs[j] = z0[k * 100 + j];
    tzs[j] = tz0[k * 100 + j];
  }
  __syncthreads();
  if (j < 100) {
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W0 = mw + (net * 3 + 0) * 10000;
      float a = mb[(net * 3 + 0) * 100 + j], t = 0.f;
      for (int i = 0; i < 100; ++i) {
        a = fmaf(zs[i], W0[i * 100 + j], a);
        t = fmaf(tzs[i], W0[i * 100 + j], t);
      }
      us[net][j] = 0.5f * (a + fabsf(a));
      tus[net][j] = t * rect_grad(a);
    }
  }
  __syncthreads();
  if (j < 100) {
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W0 = mw + (net * 3 + 0) * 10000;
      float a = mb[(net * 3 + 0) * 100 + j], t = 0.f;
      for (int i = 0; i < 100; ++i) {
        a = fmaf(us[net][i], W0[i * 100 + j], a);
        t = fmaf(tus[net][i], W0[i * 100 + j], t);
      }
      hs[net][j] = 0.5f * (a + fabsf(a));
      ths[net][j] = t * rect_grad(a);
    }
  }
  __syncthreads();
  if (j < 100) {
    float o[2], to[2];
#pragma unroll
    for (int net = 0; net < 2; ++net) {
      const float* W1 = mw + (net * 3 + 1) * 10000;
      const float* Wd = mw + (net * 3 + 2) * 10000;
      float a = mb[(net * 3 + 1) * 100 + j] + mb[(net * 3 + 2) * 100 + j];
      float a1 = 0.f, a2 = 0.f, t1 = 0.f, t2 = 0.f;
      for (int i = 0; i < 100; ++i) {
        a1 = fmaf(hs[net][i], W1[i * 100 + j], a1);
        a2 = fmaf(us[net][i], Wd[i * 100 + j], a2);
        t1 = fmaf(ths[net][i], W1[i * 100 + j], t1);
        t2 = fmaf(tus[net][i], Wd[i * 100 + j], t2);
      }
      o[net] = a + a1 + a2;
      to[net] = t1 + t2;
    }
    const float e = expf(o[1]);
    const float z = (zs[j] - o[0]) / e;
    tz[k * 100 + j] = (tzs[j] - to[0]) / e - z * to[1];
  }
}

// th (n,256) float32 = the tangent [t_mu | t_ls | 0] of the encoder head (BatchNorm scale applied, no shift), head the
// forward's: t_z_iaf = t_mu (+ exp(logsigma) eps t_ls) -- the transpose of enc_vjp_seed_kernel's map; eps is a constant.
__global__ void sample_tangent_kernel(const float* __restrict__ head, const float* __restrict__ eps, const float* __restrict__ th,
                                      float* __restrict__ tz, int n) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 100) return;
  const int k = i / 100, j = i % 100;
  float v = th[k * 256 + j];
  if (eps) v = fmaf(expf(head[k * 256 + 100 + j]) * eps[i], th[k * 256 + 100 + j], v);
  tz[i] = v;
}

// head (n,256) float32 = [mu | logsigma | 0] after BatchNorm; z_iaf = mu (+ exp(logsigma) eps) (sample_kernel).
// out (n,256) split planes: d(pre-BN head) = [dz scale_mu | dz exp(logsigma) eps scale_ls | 0].
__global__ void enc_vjp_seed_kernel(const float* __restrict__ head, const float* __restrict__ eps, const float* __restrict__ dz,
                                    const float* __restrict__ scale, __nv_bfloat16* __restrict__ out, long long plane, int n) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 256) return;
  const int k = i / 256, j = i % 256;
  float v = 0.f;
  if (j < 100) v = dz[k * 100 + j] * scale[j];
  else if (j < 200 && eps) v = dz[k * 100 + j - 100] * expf(head[k * 256 + j]) * eps[k * 100 + j - 100] * scale[j];
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  out[i] = hi;
  out[plane + i] = lo;
}

// g (n,1024) float32 = d loss / d enc_fc1 output; f1 (n,1024) split planes = that output (columns >= 1000 are zero).
//   rectify (IAN.py:118): derivative 1 where f1 > 0, else 0 (f1 = 0 covers pre-activations <= 0; an exact 0 would get 1/2
//   in Theano, which float inputs do not reach);  elu (IAN_simple.py:121): 1 where f1 > 0, else exp(u) = f1 + 1.
__global__ void enc_fc1_bwd_kernel(const float* __restrict__ g, const __nv_bfloat16* __restrict__ f1, long long f1_plane,
                                   const float* __restrict__ scale, int elu, __nv_bfloat16* __restrict__ out, long long plane,
                                   int n) {
  pdl_trigger();
  pdl_wait();                                           // tapgemm.h: PDL
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 1024) return;
  const float y = __bfloat162float(f1[i]) + __bfloat162float(f1[f1_plane + i]);
  const float d = y > 0.f ? 1.f : (elu ? y + 1.f : 0.f);
  __nv_bfloat16 hi, lo;
  split_bf16(g[i] * d * scale[i % 1024], hi, lo);
  out[i] = hi;
  out[plane + i] = lo;
}

// out[t'][c][r] = in[flip ? ntiles-1-t' : t'][r][c] over both planes (a bf16 hi|lo split is per element: bit-exact)
__global__ void permute_tiles_kernel(const __nv_bfloat16* __restrict__ in, long long in_plane, __nv_bfloat16* __restrict__ out,
                                     int ntiles, int R, int C, int flip) {
  const long long total = (long long)ntiles * R * C;
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total; o += (long long)gridDim.x * blockDim.x) {
    const long long t = o / ((long long)R * C);
    const int rem = (int)(o - t * R * C);
    const int c = rem / R, r = rem % R;
    const long long src = ((flip ? ntiles - 1 - t : t) * R + r) * (long long)C + c;
    out[o] = in[src];
    out[total + o] = in[in_plane + src];
  }
}

}  // namespace

int launch_made_iaf_bwd(const float* z0, const float* mw, const float* mb, const float* dz, float* dzi, int n, cudaStream_t st) {
  if (launch_pdl(made_iaf_bwd_kernel, dim3(n), dim3(128), 0, st, z0, mw, mb, dz, dzi, n) != cudaSuccess) return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_made_iaf_tangent(const float* z0, const float* tz0, const float* mw, const float* mb, float* tz, int n, cudaStream_t st) {
  if (launch_pdl(made_iaf_tangent_kernel, dim3(n), dim3(128), 0, st, z0, tz0, mw, mb, tz, n) != cudaSuccess) return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_sample_tangent(const float* head, const float* eps, const float* th, float* tz, int n, cudaStream_t st) {
  if (launch_pdl(sample_tangent_kernel, dim3((n * 100 + 255) / 256), dim3(256), 0, st, head, eps, th, tz, n) != cudaSuccess)
    return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_enc_vjp_seed(const float* head, const float* eps, const float* dz, const float* scale, __nv_bfloat16* out,
                        long long plane, int n, cudaStream_t st) {
  if (launch_pdl(enc_vjp_seed_kernel, dim3((n * 256 + 255) / 256), dim3(256), 0, st, head, eps, dz, scale, out, plane, n) != cudaSuccess)
    return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_enc_fc1_bwd(const float* g, const __nv_bfloat16* f1, long long f1_plane, const float* scale, int elu,
                       __nv_bfloat16* out, long long plane, int n, cudaStream_t st) {
  if (launch_pdl(enc_fc1_bwd_kernel, dim3((n * 1024 + 255) / 256), dim3(256), 0, st, g, f1, f1_plane, scale, elu, out, plane, n) != cudaSuccess)
    return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_permute_tiles(const __nv_bfloat16* in, long long in_plane, __nv_bfloat16* out, int ntiles, int R, int C, int flip,
                         cudaStream_t st) {
  permute_tiles_kernel<<<1024, 256, 0, st>>>(in, in_plane, out, ntiles, R, C, flip);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ian
