// edge.h -- launchers of the HBM-bound end kernels and glue (see edge_kernels.cu).
#pragma once
#include "tapgemm.h"

namespace ian {
// every launcher returns the number of kernels launched (1) or <0 on a launch error
int launch_conv1(const float* x, const float* wt, const float* bias, __nv_bfloat16* out, long long plane, int n,
                 cudaStream_t st);
int launch_dec_out(const __nv_bfloat16* h3, long long plane, const float* wt, float* xhat, int n, cudaStream_t st);
// enc_conv1's adjoint for the encoder VJP: dec_out's kernel body with an identity epilogue on the conv1 gradient planes e1
// (n,32,32,128) and the tap-flipped conv1 weights wt[t][o][c(4)] = W[o][c][24-t] -> dx (n,3,64,64) float32
int launch_conv1_bwd(const __nv_bfloat16* e1, long long plane, const float* wt, float* dx, int n, cudaStream_t st);
// the rest of the encoder VJP's small kernels (enc_vjp.cu)
int launch_made_iaf_bwd(const float* z0, const float* mw, const float* mb, const float* dz, float* dzi, int n, cudaStream_t st);
int launch_enc_vjp_seed(const float* head, const float* eps, const float* dz, const float* scale, __nv_bfloat16* out,
                        long long plane, int n, cudaStream_t st);
int launch_enc_fc1_bwd(const float* g, const __nv_bfloat16* f1, long long f1_plane, const float* scale, int elu,
                       __nv_bfloat16* out, long long plane, int n, cudaStream_t st);
int launch_permute_tiles(const __nv_bfloat16* in, long long in_plane, __nv_bfloat16* out, int ntiles, int R, int C, int flip,
                         cudaStream_t st);
// encoder JVP (ian_encode_jvp_*).  enc_conv1's tangent on the SIMT path: conv1_kernel's body on the tangent image v, no bias,
// times LeakyRectify' from the sign of the stored a1 planes -> the tangent planes of a1 (edge_kernels.cu).  Then (enc_vjp.cu)
// the sample tangent th (n,256) [t_mu | t_ls] -> t_z_iaf (n,100), and forward mode through the MADE/IAF flow from the
// forward's z0 and the tangent tz0 -> tz (n,100).
int launch_conv1_tangent(const float* v, const float* wt, const __nv_bfloat16* a1, __nv_bfloat16* out, long long plane, int n,
                         cudaStream_t st);
int launch_sample_tangent(const float* head, const float* eps, const float* th, float* tz, int n, cudaStream_t st);
int launch_made_iaf_tangent(const float* z0, const float* tz0, const float* mw, const float* mb, float* tz, int n, cudaStream_t st);
int launch_sample(const float* head, const float* eps, float* z, __nv_bfloat16* zp, long long zplane, int n,
                  cudaStream_t st);
int launch_z_to_planes(const float* z, __nv_bfloat16* zp, long long zplane, int n, cudaStream_t st);
// loss seed (box form; or, with dxhat != NULL, a caller's (n,3,64,64) cotangent over the whole frame) + dec_out backward
int launch_brush_seed_bwd(const float* xhat, const int32_t* boxes, const float* target, int target_is_frame, const float* dxhat,
                          const float* wt, const float* scale3, const __nv_bfloat16* h3, __nv_bfloat16* d3,
                          long long plane, int n, cudaStream_t st);
// the dense seed of the parameter VJP: d3 exactly as launch_brush_seed_bwd(dxhat) writes it, plus the seed image
// dx_hat * (1 - x_hat^2) (n,3,64,64) for dec_out's weight gradient and dL/dh3 before mask and scale (split planes, d3's
// geometry) for bnorm_dc3
int launch_brush_param_seed_bwd(const float* xhat, const float* dxhat, const float* wt, const float* scale3,
                                const __nv_bfloat16* h3, __nv_bfloat16* d3, long long plane, float* seed_out,
                                __nv_bfloat16* dh3, int n, cudaStream_t st);
// parameter-VJP reductions (param_vjp.cu); part: per-chunk partial sums, sized by decout_wgrad_chunks / bn_param_chunks
int decout_wgrad_chunks(int n);                         // part: chunks * 25 * 384 floats
int bn_param_chunks(int C, long long R);                // part: chunks * 2 * C floats
int launch_decout_wgrad(const float* seed, const __nv_bfloat16* h3, long long plane, int n, float* part, float* out,
                        int accumulate, cudaStream_t st);
int launch_bn_param_bwd(const __nv_bfloat16* dh, long long dh_plane, const __nv_bfloat16* h, const __nv_bfloat16* x,
                        long long x_plane, const float* mean, const float* istd, int C, long long R, int fc2, float* part,
                        float* dbeta, float* dgamma, int accumulate, cudaStream_t st);
int launch_brush_update(const float* gpad, const int32_t* boxes, float weight, float* g_out, float* z,
                        __nv_bfloat16* zp, long long zplane, int n, cudaStream_t st);
// NPE photo-mode blend + display upsample after a stroke (NPE.py:107-118, 218-231)
int launch_npe_blend(const float* xhat, const uint8_t* recon, const float* error, uint8_t* im, uint8_t* display, cudaStream_t st);
// full IAN: MADE+IAF latent flow and the autoregressive RGB-Beta head
int launch_made_iaf(const float* z0, const float* mw, const float* mb, float* z, __nv_bfloat16* zp, long long zplane, int n,
                    cudaStream_t st);
int launch_head_gather(const float* tt, int tt_is_bf16, const int* taps, int ntaps, float* ha, int n, cudaStream_t st);
int launch_rgb_beta_head(const float* ha, int ha_planar, float* rg, const int* taps, const float* wgb, const float* wbb, int ntaps,
                         float* xhat, float* bsave /*nullable*/, int n, cudaStream_t st);
// brush gradient through the RGB-Beta head: seed over the box (or, with dxhat != NULL, a caller's cotangent over the whole
// frame) and the Beta backward into dpre (n,64,64,8); then the autoregressive backward and the im2col operand a2
// (n,64,64,256 split planes) of the dense backward GEMM (see edge_kernels.cu)
int launch_head_bwd_seed(const float* xhat, const float* rg, const float* bsave, const int32_t* boxes, const float* target,
                         int target_is_frame, const float* dxhat, float* dpre, int n, cudaStream_t st);
int launch_head_bwd(const float* rg, const int* taps, const float* wgb, const float* wbb, int ntaps, float* dpre,
                    __nv_bfloat16* a2, long long a2_plane, int n, cudaStream_t st);
// decoder JVP (ian_decode_jvp_*).  Through the RGB-Beta head: tha = the three MDC convolutions of h4's tangent (ha's
// layouts), rg / bsave the primal sigmoids of the forward -> tangent sigmoids trg (n,64,64,4) and dx_hat (n,3,64,64).
// Through IAN_simple's dec_out (SIMT): the tangent planes t3 of h3 and the primal x_hat -> dx_hat = conv(t3) * (1 - x_hat^2).
int launch_rgb_beta_head_jvp(const float* tha, int tha_planar, const float* rg, const float* bsave, float* trg, const int* taps,
                             const float* wgb, const float* wbb, int ntaps, float* dxhat, int n, cudaStream_t st);
int launch_dec_out_jvp(const __nv_bfloat16* t3, long long plane, const float* wt, const float* xhat, float* dxhat, int n,
                       cudaStream_t st);
// RGB-Beta head on the tensor-core path (head_tc.cu): dense GEMM per (image, conv) + on-chip tap gather -> ha [n][6][4096]
// (the autoregressive sigmoid / Beta part stays the three per-pixel kernels of edge_kernels.cu)
struct HeadMaps;
HeadMaps* head_build_maps(const __nv_bfloat16* fh4, long long fh4_plane, int n_img, const __nv_bfloat16* wt, long long wt_plane,
                          char* err, int errlen);
void head_free_maps(HeadMaps*);
int launch_head_tc(const HeadMaps* maps, int passes, float* ha, int n, cudaStream_t st);
// enc_conv1 on the tensor-core path (conv1_tc.cu): thread-built im2col tile + wgmma
struct Conv1Maps;
struct Conv1OutMap;
// wt: three blocks of [128 cout][64 k] bf16 (hi k<64 | lo k<64 | tail: hi k 64..79, lo k 64..79, zeros)
Conv1Maps* conv1_build_maps(const __nv_bfloat16* wt, char* err, int errlen);
void conv1_free_maps(Conv1Maps*);
// per plan: the TMA-store view of the a1 activation planes the kernel writes
Conv1OutMap* conv1_build_out_map(__nv_bfloat16* out, long long plane, int n, char* err, int errlen);
void conv1_free_out_map(Conv1OutMap*);
int launch_conv1_tc(const Conv1Maps* maps, const Conv1OutMap* omap, const float* x, const float* bias, int n, cudaStream_t st);
// encoder JVP: enc_conv1's tangent on the tensor cores -- conv1_tc's GEMM on the tangent image v, no bias, LeakyRectify' from
// the sign of the stored a1 (hi plane) -> the planes omap was built on
int launch_conv1_tangent_tc(const Conv1Maps* maps, const Conv1OutMap* omap, const float* v, const __nv_bfloat16* a1, int n,
                            cudaStream_t st);
// dec_out on the tensor-core path (decout_tc.cu)
struct DecOutMaps;
DecOutMaps* decout_build_maps(const __nv_bfloat16* h3, long long h3_plane, int n_img, const __nv_bfloat16* wt,
                              long long wt_plane, char* err, int errlen);
void decout_free_maps(DecOutMaps*);
// dsts[0..ndst): destination base pointers (1 = local only; >1 = every rank's gather buffer incl. peers)
int launch_dec_out_tc(const DecOutMaps* maps, float* const* dsts, int ndst, int n, cudaStream_t st);
// enc_conv1's adjoint on the tensor-core path: decout_tc's kernel body with an identity epilogue; maps built by
// decout_build_maps on the conv1 gradient planes e1 and the [2][80][128] planes of rows tap*3 + c = W1[o][c][24 - tap]
int launch_conv1_bwd_tc(const DecOutMaps* maps, float* dx, int n, cudaStream_t st);
// decoder JVP on the tensor-core path: decout_tc's GEMM + col2im on the tangent planes of h3 (maps built by decout_build_maps
// on them, with dec_out's weights), epilogue dx_hat = y * (1 - x_hat^2) from the primal x_hat
int launch_dec_out_jvp_tc(const DecOutMaps* maps, const float* xhat, float* dxhat, int n, cudaStream_t st);
// latent fit (gn_kernels.cu, ian_decode_gauss_newton_* / ian_fit_latent_*).  The Levenberg-Marquardt constants, fixed:
// lambda starts at 1e-3, is divided by 10 on an accepted step (not below 1e-7) and multiplied by 10 on a rejected one (not
// above 1e10); the damping is lambda * diag(max(A_ii, 1e-9 * max_j A_jj)).
constexpr double kGnLambda0 = 1e-3, kGnLambdaMin = 1e-7, kGnLambdaMax = 1e10, kGnLambdaFactor = 10.0, kGnDampFloor = 1e-9;
// Thread 0 of sample k's accept CTA, with et the objective at the trial (init: at the start): init sets e and lambda;
// otherwise the step is taken when it was solved (ok) and et < e, e <- et and lambda <- max(lambda / 10, min), else
// lambda <- min(10 lambda, max).  loss[k * ldl + col] (nullable) = e / 12288 after the decision.  Returns whether the
// step is taken; every accept kernel decides through this.
__device__ __forceinline__ int gn_decide(int init, double et, const int* ok, double* e, double* lam, float* loss, long long ldl,
                                         int col, int k) {
  int take = 0;
  if (init) {
    e[k] = et;
    lam[k] = kGnLambda0;
  } else {
    take = ok[k] && et < e[k];
    if (take) {
      e[k] = et;
      lam[k] = fmax(lam[k] / kGnLambdaFactor, kGnLambdaMin);
    } else {
      lam[k] = fmin(lam[k] * kGnLambdaFactor, kGnLambdaMax);
    }
  }
  if (loss) loss[(size_t)k * ldl + col] = (float)(e[k] / 12288.0);
  return take;
}
size_t gn_part_doubles();                              // the Gram's chunk partials, per JVP pass
// z (100) -> zrep (100,100), every row z
int launch_gn_replicate(const float* z, float* zrep, cudaStream_t st);
// J (100,12288) float32, x_hat and x (12288) -> A (100,100), g (100), e (nullable) float64, via part (gn_part_doubles())
int launch_gn_gram(const float* J, const float* xh, const float* x, double* part, double* A, double* g, double* e,
                   cudaStream_t st);
// per sample k < n: A (n,100,100), g (n,100), lambda (n) float64, z (n,100) -> z_trial (n,100), ok (n): 0 = rejected step
int launch_gn_solve(const double* A, const double* g, const double* lam, const float* z, float* zt, int* ok, int n,
                    cudaStream_t st);
// per sample: e_trial from x_hat_trial and x (n,12288), then accept or reject (init: set e, lambda from the start) and
// loss[k * ldl + col] (nullable) = e / 12288
int launch_gn_accept(int init, const float* xht, const float* x, float* xh, double* e, double* lam, float* z, const float* zt,
                     const int* ok, float* loss, long long ldl, int col, int n, cudaStream_t st);
// the masked fit under the prior (ian_map_gauss_newton_* / ian_fit_latent_map_*): launch_gn_gram and launch_gn_accept with
// the pixel weight w (nullable: all ones; w == 0 pixels skipped) and the prior weight beta on the fit-space point u (100):
// A = J^T W J + beta I, g = J^T W r + beta u, e = r^T W r + beta |u|^2
int launch_map_gram(const float* J, const float* xh, const float* x, const float* w, double beta, const float* u, double* part,
                    double* A, double* g, double* e, cudaStream_t st);
int launch_map_accept(int init, const float* xht, const float* x, const float* w, double beta, float* xh, double* e, double* lam,
                      float* u, const float* ut, const int* ok, float* loss, long long ldl, int col, int n, cudaStream_t st);
// the robust fit (ian_robust_gauss_newton_* / ian_fit_latent_robust_*): launch_map_gram and launch_map_accept with
// omega = w rho'(r^2) as the pixel weight and E = sum w rho(r^2) + beta |u|^2, kind kRobustHuber or kRobustCauchy (the
// header's IAN_ROBUST_*), dl the per-sample scale delta (robust_gram: the one sample's).  The automatic scale is
// max(m c, kRobustScaleFloor) with m the lower median of float32 |r| over the weighted pixels and c the loss's 95 %-efficiency
// constant times 1.4826 (the MAD's Gaussian consistency); the floor is half an 8-bit level on [-1, 1].
constexpr int kRobustHuber = 1, kRobustCauchy = 2;
constexpr double kRobustHuberC = 1.345 * 1.4826, kRobustCauchyC = 2.3849 * 1.4826, kRobustScaleFloor = 1.0 / 255.0;
int launch_robust_gram(const float* J, const float* xh, const float* x, const float* w, int kind, const double* dl, double beta,
                       const float* u, double* part, double* A, double* g, cudaStream_t st);
int launch_robust_accept(int init, const float* xht, const float* x, const float* w, double beta, int kind, const double* dl,
                         float* xh, double* e, double* lam, float* u, const float* ut, const int* ok, float* loss, long long ldl,
                         int col, int n, cudaStream_t st);
// dl (n) from x_hat and x (n,12288), w (nullable)
int launch_robust_scale(const float* xh, const float* x, const float* w, int kind, double* dl, int n, cudaStream_t st);
// out (n,12288) = rho'(r^2) per element, 0 where w == 0
int launch_robust_outliers(const float* xh, const float* x, const float* w, int kind, const double* dl, float* out, int n,
                           cudaStream_t st);
// the IAN's introspection features and the fit under its feature-wise loss (feat_kernels.cu; ian_introspect_*,
// ian_feature_gauss_newton_*, ian_fit_latent_features_*): layer l = 0..3 is enc_conv{l+1}'s output a{l+1}, (32 >> l)^2
// pixels of 128 << l channels, M_l elements per image
constexpr int kFeatTotal = 245760;
__host__ __device__ __forceinline__ long long feat_m(int l) { return 131072LL >> l; }
struct FeatLayers {           // per layer: split planes (tan, plane) and float32 NHWC features (cur, tgt)
  const __nv_bfloat16* tan[4];
  long long plane[4];
  float* cur[4];
  const float* tgt[4];
};
struct FeatWeights {          // E = a |r|^2 + sum_l c[l] |r_l|^2
  double a;
  double c[4];
};
size_t feat_part_doubles();   // the feature Gram's chunk partials, per sample
// layer `layer` of n images: split planes (hi only when passes == 1) -> float32, NCHW when nchw, else NHWC
int launch_feat_store(const __nv_bfloat16* p, long long plane, int passes, int layer, int n, float* out, int nchw,
                      cudaStream_t st);
// one sample: t.tan = the 100 tangent rows of every layer (plan of 100), t.cur / t.tgt = the sample's features ->
// A (100,100), g (100), e (nullable) = sum_l c[l] [J_l | r_l]^T [J_l | r_l] (feats == 0: no such terms, t unread), plus
// c.a times what A, g, e hold when pixel != 0 (the pixel Gram of launch_gn_gram)
int launch_feat_gram(const FeatLayers& t, const FeatWeights& c, int feats, int passes, int pixel, double* part, double* A,
                     double* g, double* e, cudaStream_t st);
// launch_gn_accept on E: f.tan = the trial's feature planes (plan of n), f.tgt the target's and f.cur the current features
// (n samples each, float32 NHWC); the start and every accepted step copy the trial's features into f.cur.  feats == 0:
// no feature terms; c.a == 0: no pixel term
int launch_feat_accept(int init, const float* xht, const float* x, const FeatLayers& f, const FeatWeights& c, int feats,
                       int passes, float* xh, double* e, double* lam, float* z, const float* zt, const int* ok, float* loss,
                       long long ldl, int col, int n, cudaStream_t st);
// the features' vector-Jacobian product (ian_introspect_vjp_*): per layer l the cotangent c[l] (n, 128 << l, 32 >> l,
// 32 >> l) float32 NCHW (nullptr: not supplied) -> split planes NHWC at out[l].  Layer `deep` is the chain's seed:
// r * scale[ch] * (hi(mask) > 0 ? 1 : 0.2) with r = c as a backward GEMM reads it as `res` (hi + lo; hi when passes == 1),
// the ACT_MASK epilogue on a_deep with a zero accumulator (scale nullptr: 1).  Its lo plane is written only when deep_lo
// is set: exactly when the backward GEMM landing on that layer writes it (float32 mode, or a split-K finalize), since
// those planes are the encoder VJP's and a later call may read them.  The others are stored as they are, for the backward
// GEMMs' `res`.  One launch covers every supplied layer.
struct FeatCotangents {
  const float* c[4];
  __nv_bfloat16* out[4];
  long long plane[4];
  int deep, deep_lo;
  const __nv_bfloat16* mask;
  const float* scale;
};
int launch_feat_cotangent(const FeatCotangents& c, int passes, int n, cudaStream_t st);
// the discriminator head l_discrim (disc_kernels.cu; ian_discriminate_*): its MinibatchLayer has kDiscKernels kernels of 5
// dimensions on the 1024 pooled channels of a4, its dense layer 1024 + kDiscKernels -> U (1 or kDiscMaxUnits) units
constexpr int kDiscKernels = 500, kDiscDims = 5, kDiscMaxUnits = 3;
// a4 (split planes of n images; hi only when passes == 1) -> pooled (n,1024), the mean over the 4 x 4 pixels
int launch_disc_pool(const __nv_bfloat16* a4, long long plane, int passes, int n, float* out, cudaStream_t st);
// in (n,1524) = [pool | f], W (1524,U) -> logits (n,U) and p (n,U, nullable) = sigmoid (U = 1) or softmax (U = 3)
int launch_disc_head(const float* in, const float* W, int U, int n, float* logits, float* p, cudaStream_t st);
// g (n,1524) = dlogits (n,U) W^T
int launch_disc_head_bwd(const float* dlogits, const float* W, int U, int n, float* g, cudaStream_t st);
// c4 (n,1024,4,4) NCHW = dpool (n,1024) / 16 at every pixel
int launch_disc_cotangent(const float* dpool, int n, float* c4, cudaStream_t st);
// the batch-statistics BatchNorm stacks (ian_discriminate_train*, ian_decode_train*): whole-call float32 NHWC (n, hw, c).
// part: [n][2][c] doubles of per-image Σu, Σu·v; sums[2][c] their image-ordered totals; count > 0 (the forward): also mean_f,
// inv_std_f (eps inside the root)
int launch_nhwc_bn_sums(const float* u, const float* v, int n, int hw, int c, double count, float eps, double* part, double* sums,
                        float* mean_f, float* inv_std_f, cudaStream_t st);
// x (total elements, channel fastest) -> fmaf(act_abs, |y|, act_lin y), y = (x - mean) (gamma inv_std) + beta, as split planes
// (hi only if passes == 1)
int launch_nhwc_bn_act(const float* x, long long total, int c, const float* mean, const float* inv_std, const float* gamma,
                       const float* beta, float act_abs, float act_lin, int passes, __nv_bfloat16* out, long long plane,
                       cudaStream_t st);
// BatchNorm backward: coef[4][c] from the forward's sums and the backward's (Σdy, Σdy·x), then dx as split planes
int launch_nhwc_bn_coef(const double* fsum, const double* bsum, double count, float eps, const float* gamma, int c, double* coef,
                        cudaStream_t st);
int launch_nhwc_bn_dx(const float* x, const float* dy, long long total, int c, const double* coef, int passes, __nv_bfloat16* out,
                      long long plane, cudaStream_t st);
// dy4 (n,4,4,1024) = dpool / 16 * lrelu'(y4), y4 the batch-normalised enc_conv4 of x4
int launch_disc_train_cotangent(const float* dpool, const float* x4, int n, const float* mean, const float* inv_std,
                                const float* gamma, const float* beta, float* dy, cudaStream_t st);
// the IAN_simple decoder in training mode (ian_decode_train*): dy (float32) = (hi + lo of the split planes dh) * (y > 0), y the batch-normalised x
int launch_dec_train_dy(const __nv_bfloat16* dh, long long plane, const float* x, long long total, int c, const float* mean,
                        const float* inv_std, const float* gamma, const float* beta, float* dy, cudaStream_t st);
// d beta, d gamma (nullable each) from the forward's and the backward's [2][c] sums; fc2: columns in bnorm_dec_fc2's library
// order, written at their reference feature
int launch_dec_bn_grads(const double* fsum, const double* bsum, double count, float eps, int c, int fc2, float* dbeta,
                        float* dgamma, cudaStream_t st);
// [2][total] statistics with bnorm_dec_fc2's first fc2_cols columns moved to their reference feature
int launch_dec_stats_out(const float* in, int total, int fc2_cols, float* out, cudaStream_t st);
// signal + wait kernels of the peer-memory barrier (flag_ptrs[r] = rank r's flag array, int[8])
int launch_peer_barrier(float* const* flag_ptrs, int world, int rank, int epoch, cudaStream_t st);
// training-mode pieces (train_kernels.cu): BatchNorm batch statistics / normalisation, MinibatchLayer forward
size_t bn_workspace_bytes(int c);
int launch_bn_batch_stats(const float* x, int n, int c, int hw, double* sum, double* sumsq, void* ws, cudaStream_t st);
int launch_bn_train_normalize(const float* x, int n, int c, int hw, const double* sum, const double* sumsq, double count,
                              const float* gamma, const float* beta, float eps, float alpha, float* running_mean,
                              float* running_inv_std, float* y, void* ws, cudaStream_t st);
size_t mb_workspace_bytes(int n, int K, int P);
int launch_minibatch_discrim(const float* x, int n, int d, const float* theta, const float* lws, const float* b, int K, int P,
                             float* out, void* ws, cudaStream_t st);
// their reverse mode: BatchNorm backward sums (+ local dgamma / dbeta) and dx; MinibatchLayer dx, dtheta, dlws, db
int launch_bn_backward_sums(const float* x, const float* dy, int n, int c, int hw, const double* sum, const double* sumsq, double count,
                            float eps, double* sum_dy, double* sum_dyx, float* dgamma, float* dbeta, void* ws, cudaStream_t st);
int launch_bn_backward_dx(const float* x, const float* dy, int n, int c, int hw, const double* sum, const double* sumsq, double count,
                          const double* sum_dy, const double* sum_dyx, const float* gamma, float eps, float* dx, void* ws, cudaStream_t st);
size_t mb_bwd_workspace_bytes(int n, int d, int K, int P);
int launch_minibatch_discrim_bwd(const float* x, int n, int d, const float* theta, const float* lws, int K, int P, const float* g,
                                 float* dx, float* dtheta, float* dlws, float* db, void* ws, cudaStream_t st);
// pipelined all-gather: copy this rank's decoded shard (src, n_floats) into every peer's gather buffer from a small
// side-stream kernel + free/pushed flag handshake (see decout_tc.cu); returns after enqueueing push + wait kernels
int launch_peer_push(const float* src, float* const* dsts, float* const* flag_ptrs, long long n_floats, int world, int rank,
                     int step, int ctas, cudaStream_t st);
}  // namespace ian
