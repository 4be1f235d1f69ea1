// ian_api.cu -- C-ABI of libian_b200.so (include/ian_b200.h): handle, weight preparation, per-batch
// plans (activation buffers in HBM + tap-GEMM descriptors + TMA maps) and the layer schedules of the
// IAN_simple graph (reference IAN_simple.py:56-241) for encode, decode, brush gradient and edit loop.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include <cuda.h>

#include "../../include/ian_b200.h"
#include "edge.h"
#include "tapgemm.h"

using namespace ian;

namespace {

thread_local std::string g_create_error;

// ------------------------------------------------------------------------------------------------
// host-side bf16 helpers (round-to-nearest-even), independent of device headers
// ------------------------------------------------------------------------------------------------
inline uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN
  const uint32_t r = 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)((u + r) >> 16);
}
inline float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
// float32 w as the bf16 pair hi + lo that the 3-pass tensor-core kernels multiply
inline void split_hi_lo(float w, uint16_t& hi, uint16_t& lo) {
  hi = f2bf(w);
  lo = f2bf(w - bf2f(hi));
}

struct HostParam {
  std::vector<int64_t> shape;
  std::vector<float> data;
};

struct ParamSpec {
  const char* name;
  int ndim;
  int64_t shape[4];
};

// reference checkpoint names / shapes (IAN_simple.py layer names; SURVEY Appendix A)
const ParamSpec kSimpleWeights[] = {
    {"enc_conv1.W", 4, {128, 3, 5, 5}},    {"enc_conv1.b", 1, {128}},
    {"enc_conv2.W", 4, {256, 128, 5, 5}},  {"enc_conv3.W", 4, {512, 256, 5, 5}},
    {"enc_conv4.W", 4, {1024, 512, 5, 5}}, {"enc_fc1.W", 2, {16384, 1000}},
    {"enc_mu.W", 2, {1000, 100}},          {"enc_logsigma.W", 2, {1000, 100}},
    {"l_dec_fc2.W", 2, {100, 16384}},      {"dec_conv1.W", 4, {1024, 512, 5, 5}},
    {"dec_conv2.W", 4, {512, 256, 5, 5}},  {"dec_conv3.W", 4, {256, 128, 5, 5}},
    {"dec_out.W", 4, {128, 3, 5, 5}},
};
struct BnSpec { const char* name; int64_t c; };
const BnSpec kSimpleBn[] = {{"bnorm2", 256},       {"bnorm3", 512},     {"bnorm4", 1024},  {"bnorm_enc_fc1", 1000},
                            {"mu_bnorm", 100},     {"ls_bnorm", 100},   {"bnorm_dec_fc2", 16384},
                            {"bnorm_dc1", 512},    {"bnorm_dc2", 256},  {"bnorm_dc3", 128}};
const char* kBnFields[] = {"beta", "gamma", "mean", "inv_std"};

struct Spec { std::string name; std::vector<int64_t> shape; };

void add_bn(std::vector<Spec>& v, const std::string& name, int64_t c) {
  for (const char* f : kBnFields) v.push_back({name + "." + f, {c}});
}
void add_mdcl(std::vector<Spec>& v, const std::string& name, int64_t F, int64_t C, std::initializer_list<int> scales) {
  v.push_back({name + "W", {F, C, 3, 3}});
  v.push_back({name + "_coeff_base", {F}});
  for (int s : scales) v.push_back({name + (s == 0 ? std::string("_coeff_1x1") : "_coeff_" + std::to_string(s)), {F}});
}
void add_mdblock(std::vector<Spec>& v, const std::string& name, int64_t F, std::initializer_list<int> scales) {
  add_mdcl(v, name, F, F, scales);
  add_mdcl(v, name + "2", F, F, scales);
  add_bn(v, name + "bnorm0", F); add_bn(v, name + "bnorm1", F); add_bn(v, name + "bnorm2", F);
}

// parameter names / shapes of a model kind, in the reference's checkpoint naming (GANcheckpoints.py:11-30)
std::vector<Spec> spec_list(int kind) {
  std::vector<Spec> v;
  if (kind == IAN_MODEL_SIMPLE) {
    for (const auto& s : kSimpleWeights) v.push_back({s.name, std::vector<int64_t>(s.shape, s.shape + s.ndim)});
    for (const auto& b : kSimpleBn) add_bn(v, b.name, b.c);
    return v;
  }
  // IAN.py:67-207
  for (const auto& s : kSimpleWeights) {
    const std::string n = s.name;
    if (n.rfind("enc_", 0) == 0) v.push_back({n, std::vector<int64_t>(s.shape, s.shape + s.ndim)});
  }
  for (const char* b : {"bnorm2", "bnorm3", "bnorm4"}) add_bn(v, b, b[5] == '2' ? 256 : b[5] == '3' ? 512 : 1024);
  add_bn(v, "bnorm_enc_fc1", 1000); add_bn(v, "mu_bnorm", 100); add_bn(v, "ls_bnorm", 100);
  for (const char* m : {"l_IAF_mu", "l_IAF_ls"})
    for (const char* sub : {"_input", "_output_W", "_output_D"}) {
      v.push_back({std::string(m) + sub + ".W", {100, 100}});
      v.push_back({std::string(m) + sub + ".b", {100}});
    }
  if (kind == IAN_MODEL_V1) {                             // IANv1.py:125-201
    v.push_back({"l_dec_fc2.W", {100, 16384}}); v.push_back({"l_dec_fc2.b", {16384}});
    v.push_back({"dec_conv1.W", {1024, 512, 5, 5}}); add_bn(v, "bnorm_dc1", 512);
    v.push_back({"dec_conv2.W", {512, 256, 5, 5}}); add_bn(v, "bnorm_dc2", 256);
    v.push_back({"dec_conv3.W", {256, 128, 5, 5}}); add_bn(v, "bnorm_dc3", 128);
    v.push_back({"dec_conv4.W", {128, 64, 5, 5}}); add_bn(v, "bnorm_dc4", 64);
    add_mdcl(v, "R", 2, 64, {2, 3, 4}); add_mdcl(v, "G_a", 2, 64, {2, 3, 4}); add_mdcl(v, "G_b", 2, 2, {2, 3, 4});
    add_mdcl(v, "B_a", 2, 64, {2, 3, 4}); add_mdcl(v, "B_b", 2, 4, {2, 3, 4});
    return v;
  }
  v.push_back({"l_dec_fc2.W", {100, 8192}}); v.push_back({"l_dec_fc2.b", {8192}});
  v.push_back({"dec_conv1.W", {512, 512, 5, 5}});
  add_mdblock(v, "dec_conv2a", 512, {0, 2});
  v.push_back({"dec_conv2.W", {512, 256, 5, 5}});
  add_mdblock(v, "dec_conv3a", 256, {0, 2, 3});
  v.push_back({"dec_conv3.W", {256, 128, 5, 5}});
  add_mdblock(v, "dec_conv4a", 128, {0, 2, 3});
  v.push_back({"dec_conv4.W", {128, 128, 5, 5}});
  add_bn(v, "bnorm_dc4", 128);
  add_mdcl(v, "R", 2, 128, {2, 3, 4}); add_mdcl(v, "G_a", 2, 128, {2, 3, 4}); add_mdcl(v, "G_b", 2, 2, {2, 3, 4});
  add_mdcl(v, "B_a", 2, 128, {2, 3, 4}); add_mdcl(v, "B_b", 2, 4, {2, 3, 4});
  return v;
}

const std::vector<Spec>& cached_specs(int kind) {
  static const std::vector<Spec> cache[3] = {spec_list(0), spec_list(1), spec_list(2)};
  return cache[kind];
}

enum LayerId {
  L_ENC_CONV2 = 0, L_ENC_CONV3, L_ENC_CONV4, L_ENC_FC1, L_ENC_HEAD, L_DEC_FC2, L_DEC_CONV1, L_DEC_CONV2, L_DEC_CONV3,
  L_BWD_CONV3, L_BWD_CONV2, L_BWD_CONV1, L_BWD_FC2,
  // full IAN decoder (reference IAN.py:129-207)
  F_DEC_FC2, F_DEC_CONV1, F_MD1A, F_MD1B, F_DEC_CONV2, F_MD2A, F_MD2B, F_DEC_CONV3, F_MD3A, F_MD3B, F_DEC_CONV4, F_HEAD,
  // brush gradient through the IAN.py / IANv1.py decoders (T.grad at API.py:59,64 on those graphs)
  F_BWD_HEAD, F_BWD_CONV4, F_BWD_MD3B, F_BWD_MD3A, F_BWD_CONV3, F_BWD_MD2B, F_BWD_MD2A, F_BWD_CONV2, F_BWD_MD1B, F_BWD_MD1A,
  F_BWD_CONV1, F_BWD_FC2,
  // encoder VJP (ian_encode_vjp_*): adjoints of the encoder head, enc_fc1 and enc_conv4..2, built on first use
  E_BWD_HEAD, E_BWD_FC1, E_BWD_CONV4, E_BWD_CONV3, E_BWD_CONV2,
  // decoder Jacobian-vector product (ian_decode_jvp_*): the tangent twin of every decoder forward tap-GEMM (DecoderLayers::jvp) and of the head
  // GEMM of the verification path; built on first use
  J_DEC_FC2, J_DEC_CONV1, J_DEC_CONV2, J_DEC_CONV3,
  JF_DEC_FC2, JF_DEC_CONV1, JF_MD1A, JF_MD1B, JF_DEC_CONV2, JF_MD2A, JF_MD2B, JF_DEC_CONV3, JF_MD3A, JF_MD3B, JF_DEC_CONV4,
  J_HEAD,
  // encoder Jacobian-vector product (ian_encode_jvp_*): the tangent twins of enc_conv2..4, enc_fc1 and the encoder head
  // (kEncoderJvp); built on first use
  JE_ENC_CONV2, JE_ENC_CONV3, JE_ENC_CONV4, JE_ENC_FC1, JE_ENC_HEAD,
  // the features' vector-Jacobian product (ian_introspect_vjp_*): E_BWD_CONV4..2 with a shallower feature's cotangent
  // joining before the activation derivative (res); built on first use
  IV_BWD_CONV4, IV_BWD_CONV3, IV_BWD_CONV2,
  // the training-mode discriminator (ian_discriminate_train*): enc_conv2..4 with unit scale, no shift and no activation
  // into a float32 raw buffer, and E_BWD_CONV4 / E_BWD_CONV3 with unit scale into a float32 buffer; built on first use
  DT_ENC_CONV2, DT_ENC_CONV3, DT_ENC_CONV4, DT_BWD_CONV4, DT_BWD_CONV3,
  // the IAN_simple decoder in training mode (ian_decode_train*): l_dec_fc2 and dec_conv1..3 with unit scale, no shift and no
  // activation into a float32 raw buffer, and L_BWD_CONV3..1 with unit scale into a float32 buffer; built on first use
  DD_DEC_FC2, DD_DEC_CONV1, DD_DEC_CONV2, DD_DEC_CONV3, DD_BWD_CONV3, DD_BWD_CONV2, DD_BWD_CONV1,
  L_COUNT,
  T_CONV1 = L_COUNT, T_DEC_OUT, T_BRUSH_SEED, T_CONV1_BWD,   // timing-only slots of the edge kernels (brush_seed: the
                                                        // loss-seed kernel of every decoder backward, box or dense VJP seed;
                                                        // enc_conv1_bwd: enc_conv1's adjoint, the encoder VJP's last kernel)
  T_WGRAD_FC2, T_WGRAD_CONV1, T_WGRAD_CONV2, T_WGRAD_CONV3, T_WGRAD_DEC_OUT,   // weight gradients of the parameter VJP
  T_DEC_OUT_JVP,                                        // IAN_simple's dec_out in the decoder JVP
  T_CONV1_TANGENT,                                      // enc_conv1's tangent in the encoder JVP
  T_GN_GRAM, T_GN_SOLVE,                                // the latent fit's Gram (with its chunk reduction) and LM solve
  T_MAP_GRAM,                                           // the masked fit's weighted Gram (with its reduction and the prior)
  T_FEAT_GRAM, T_FEAT_ACCEPT,                           // the feature fit's Gram over the four feature layers (with its
                                                        // reduction) and its trial reduction and accept rule
  T_FEAT_COTANGENT,                                     // the features' VJP: the cotangents' conversion to split planes
  T_ROBUST_GRAM, T_ROBUST_SCALE,                        // the robust fit's reweighted Gram (with its reduction and the
                                                        // prior) and its automatic per-sample scale
  T_DISC_POOL, T_DISC_HEAD, T_DISC_HEAD_BWD, T_DISC_MB, T_DISC_MB_BWD,   // the discriminator head: a4's pool, the dense
  T_DISC_COTANGENT,                                     // layer, their adjoints, the MinibatchLayer, and enc_conv4's cotangent
  T_DT_STATS, T_DT_NORM, T_DT_COTANGENT, T_DT_BN_BWD, T_DT_BN_DX,   // the training-mode trunk: batch statistics, normalise +
                                                        // LeakyReLU, the pool's adjoint, BatchNorm backward sums and dx
  T_DD_STATS, T_DD_NORM, T_DD_COTANGENT, T_DD_BN_BWD, T_DD_BN_DX,   // the same steps of the training-mode decoder (cotangent:
                                                        // bnorm_dc3's dy from the seed), and its BatchNorm beta / gamma
  T_DD_BN_GRADS,
  T_COUNT
};
const char* kLayerNames[T_COUNT] = {"enc_conv2", "enc_conv3", "enc_conv4", "enc_fc1", "enc_head", "l_dec_fc2", "dec_conv1",
                                    "dec_conv2", "dec_conv3", "bwd_dec_conv3", "bwd_dec_conv2", "bwd_dec_conv1", "bwd_l_dec_fc2",
                                    "full_dec_fc2", "full_dec_conv1", "dec_conv2a", "dec_conv2a2", "full_dec_conv2", "dec_conv3a", "dec_conv3a2",
                                    "full_dec_conv3", "dec_conv4a", "dec_conv4a2", "full_dec_conv4", "rgb_head",
                                    "bwd_rgb_head", "bwd_full_dec_conv4", "bwd_dec_conv4a2", "bwd_dec_conv4a", "bwd_full_dec_conv3",
                                    "bwd_dec_conv3a2", "bwd_dec_conv3a", "bwd_full_dec_conv2", "bwd_dec_conv2a2", "bwd_dec_conv2a",
                                    "bwd_full_dec_conv1", "bwd_full_dec_fc2",
                                    "bwd_enc_head", "bwd_enc_fc1", "bwd_enc_conv4", "bwd_enc_conv3", "bwd_enc_conv2",
                                    "jvp_l_dec_fc2", "jvp_dec_conv1", "jvp_dec_conv2", "jvp_dec_conv3",
                                    "jvp_full_dec_fc2", "jvp_full_dec_conv1", "jvp_dec_conv2a", "jvp_dec_conv2a2", "jvp_full_dec_conv2",
                                    "jvp_dec_conv3a", "jvp_dec_conv3a2", "jvp_full_dec_conv3", "jvp_dec_conv4a", "jvp_dec_conv4a2",
                                    "jvp_full_dec_conv4", "rgb_head_jvp",
                                    "jvp_enc_conv2", "jvp_enc_conv3", "jvp_enc_conv4", "jvp_enc_fc1", "jvp_enc_head",
                                    "introspect_bwd_enc_conv4", "introspect_bwd_enc_conv3", "introspect_bwd_enc_conv2",
                                    "disc_train_enc_conv2", "disc_train_enc_conv3", "disc_train_enc_conv4",
                                    "disc_train_bwd_enc_conv4", "disc_train_bwd_enc_conv3",
                                    "dec_train_l_dec_fc2", "dec_train_dec_conv1", "dec_train_dec_conv2", "dec_train_dec_conv3",
                                    "dec_train_bwd_dec_conv3", "dec_train_bwd_dec_conv2", "dec_train_bwd_dec_conv1",
                                    "enc_conv1", "dec_out", "brush_seed", "enc_conv1_bwd",
                                    "wgrad_l_dec_fc2", "wgrad_dec_conv1", "wgrad_dec_conv2", "wgrad_dec_conv3", "wgrad_dec_out",
                                    "dec_out_jvp", "jvp_enc_conv1", "gn_gram", "gn_solve", "map_gram",
                                    "feat_gram", "feat_accept", "feat_cotangent",
                                    "robust_gram", "robust_scale",
                                    "disc_pool", "disc_head", "disc_head_bwd", "disc_mb", "disc_mb_bwd", "disc_cotangent",
                                    "disc_train_stats", "disc_train_norm", "disc_train_cotangent", "disc_train_bn_bwd",
                                    "disc_train_bn_dx",
                                    "dec_train_stats", "dec_train_norm", "dec_train_cotangent", "dec_train_bn_bwd",
                                    "dec_train_bn_dx", "dec_train_bn_grads"};

struct DevWeights {           // one GEMM layer's B operand + epilogue vectors
  __nv_bfloat16* b = nullptr;
  long long plane = 0;
  int ntiles = 0, Cout = 0, Cin = 0;
  float* scale = nullptr;
  float* shift = nullptr;
};

struct Plan;

}  // namespace

struct ian_handle {
  int device = 0;
  int model_kind = 0;
  int path = IAN_PATH_TC;
  int passes = 3;              // 3: float32 semantics (bf16 hi|lo split); 1: plain bf16 tensor-core math
  float* sk_ws = nullptr;      // stream-K partial-sum slots + arrival flags (shared by all layers of the handle)
  int* sk_flags = nullptr;
  int sk_epoch = 0;
  int streamk = 1;             // 0: whole tiles only; 1: stream-K where the makespan test asks for it; 2: wherever eligible (tests)
  bool splitk = true;          // split-K for small-M layers (IAN_SPLITK=0: whole tiles everywhere; used by tests)
  bool coop_finalize = true;   // deep split-K layers: cooperative finalize kernel (IAN_FINALIZE8=0: one thread per output everywhere)
  bool pdl = true;             // programmatic dependent launch along the kernel chains (tapgemm.h; IAN_PDL=0 turns it off)
  bool graphs = true;          // replay small-batch host calls as CUDA graphs (IAN_GRAPHS=0 turns it off)
  bool epi_tma = true;         // plain tap-GEMM tiles leave through TMA stores (tapgemm.h; IAN_EPI_TMA=0: thread stores)
  bool capturing = false;
  bool finalized = false;
  cudaStream_t stream = nullptr;
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;   // copy streams of the pipelined host API
  std::vector<void*> host_allocs;
  // fused all-gather over NVLink peer memory (ian_gather_*): this rank's double gather buffer + flags, peers' views
  int gw = 0, grank = 0, gn = 0, gcur = 0, gepoch = 0;
  float* gbuf = nullptr;                       // [2][world][n_local][3][64][64] + flags (int[8]) at the end
  float* gpeer_buf[8] = {nullptr};             // base of every rank's allocation (peer-mapped)
  bool gconnected = false;
  float** gather_dsts = nullptr;               // non-null only inside ian_reconstruct_gather_dev
  int gather_ndst = 0;
  // pipelined gather (ian_reconstruct_gather_async_dev): side stream + per-half events
  cudaStream_t push_stream = nullptr;
  cudaEvent_t g_comp[2] = {nullptr, nullptr}, g_done[2] = {nullptr, nullptr};
  bool g_done_valid[2] = {false, false};
  int g_last = -1;                             // buffer half of the most recent async step
  int push_ctas = 32;
  int push_mode = 0;                           // 0: copy engines + stream memory ops (no SM is touched); 1: the copy kernel
  void* train_ws = nullptr;                    // workspace of the training-mode ops (grown on demand)
  size_t train_ws_bytes = 0;
  long long tickets = 0;
  struct Ticket { int id = -1, n = 0, slot = 0; };
  Ticket inflight[2];          // the two most recent pipelined requests (ian_reconstruct_submit)
  std::string err;
  int64_t launches = 0;
  std::map<std::string, HostParam> params;
  DevWeights w[L_COUNT];
  float* conv1_wt = nullptr;   // [75][128]
  float* conv1_b = nullptr;    // [128]
  __nv_bfloat16* conv1_tc_wt = nullptr;    // [3][128 cout][64 k] bf16 blocks (hi | lo | tail), k = c*25+i*5+j (75 used)
  Conv1Maps* conv1_maps = nullptr;
  float* decout_wt = nullptr;  // [25][128][4] fp32 (SIMT forward + brush backward)
  float* conv1_bwd_wt = nullptr;   // [25][128][4] fp32, W1[o][c][24-t]: enc_conv1's adjoint (built on the first encoder VJP,
                                   // with the E_BWD_* weight tiles); SIMT path
  __nv_bfloat16* conv1_bwd_tc_wt = nullptr;   // [2][80][128] bf16 planes, row = tap*3 + c, W1[o][c][24-t]; tensor-core path
  __nv_bfloat16* decout_tc_wt = nullptr;   // [2][80][128] bf16 planes, row = tap*3+co (tensor-core forward)
  std::vector<float> dec_bn[4][4];          // IAN_simple: beta, gamma, mean, inv_std of bnorm_dec_fc2, bnorm_dc1..3, kept after
                                           // finalize for ian_update_param_host
  float* dec_bn_stats[4][2] = {};          // their mean, inv_std on the device (first parameter VJP)
  float* pv_dev[13] = {};                  // the parameter VJP's gradients for the host API (first host call)
  // full IAN extras
  std::vector<int32_t> made_ordering;       // MADE input ordering (mask_generator.py:35-38); set by ian_set_made_ordering
  float *made_w = nullptr, *made_b = nullptr;   // [2][3][100][100] masked weights (in,out), [2][3][100] biases
  int* head_taps = nullptr;                 // [33][2] (dy,dx) of the scales-[2,3,4] MDC
  float *head_wgb = nullptr, *head_wbb = nullptr;   // composite G_b [33][2][2], B_b [33][2][4]
  int head_ntaps = 0;
  __nv_bfloat16* head_tc_wt = nullptr;      // fused head (head_tc.cu): [2 planes][3 convs x 80 rows][128] bf16, row = sorted tap*2 + filter
  int head_dy_start[10] = {0};              // taps sorted by row offset: taps with dy = -4 + i are [dy_start[i], dy_start[i+1])
  int head_dx[33] = {0};
  std::map<int, Plan*> plans;
  // latent fit (ian_decode_gauss_newton_*, ian_fit_latent_*; allocated on the first call): the JVP pass's identity tangents
  // and replicated latent (100,100), the Jacobian J (100,3,64,64) it writes, and the Gram's chunk partials
  float *gn_eye = nullptr, *gn_zrep = nullptr, *gn_J = nullptr;
  double* gn_part = nullptr;
  // the masked fit on IAN.py / IANv1.py: the flow's outputs on the replicated u -- z = F(u) rows, then J_F's columns (2 x 100 x 100)
  float* map_flow = nullptr;
  // the feature fit (ian_feature_gauss_newton_*, ian_fit_latent_features_*): the feature Gram's chunk partials (11.2 MB)
  double* feat_part = nullptr;
  // the discriminator head (ian_set_discriminator_param): theta, log_weight_scale, b, W on the device in the reference
  // layout, and which of the four are loaded (bit i: kDiscParams[i])
  float* disc_w[4] = {};
  int disc_set = 0;
  // ian_discriminate*'s whole-call buffers (grown to the largest batch asked for, disc_cap samples): the pooled features,
  // [pool | f], its cotangent, the pool's cotangent, the host forms' logits / p / dlogits, and one chunk's enc_conv4 cotangent
  float* disc_buf = nullptr;
  int disc_cap = 0;
  // bnorm2..4's gamma | beta (1792 + 1792 floats, uploaded with the encoder)
  float* enc_bn_gb = nullptr;
  // bnorm_dec_fc2 / bnorm_dc1..3's gamma | beta in the library's column order (2 x 17280 floats, IAN_simple, written with
  // the folded vectors)
  float* dec_bn_gb = nullptr;
  // the whole-call buffers of each batch-statistics stack (the training-mode discriminator's trunk, the IAN_simple decoder),
  // grown to the largest batch asked for, cap samples; see BnBufs
  struct { char* buf = nullptr; int cap = 0; } bn_bufs[2];
  int max_chunk = 512;
  bool timing = false;
  struct Timed { cudaEvent_t e0, e1; };
  std::vector<Timed> timed[T_COUNT];
  double time_ms[T_COUNT] = {0};
  long long time_cnt[T_COUNT] = {0};
};

namespace {

inline bool has_flow(const ian_handle* h) { return h->model_kind != IAN_MODEL_SIMPLE; }   // MADE/IAF latent + RGB-Beta head

int fail(ian_handle* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) h->err = buf; else g_create_error = buf;
  return code;
}

#define CUDA_TRY(h, expr)                                                                            \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess) return fail(h, IAN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define LAUNCH_TRY(h, expr)                                                                          \
  do {                                                                                               \
    ian::pdl_flag() = (h)->pdl && !(h)->capturing && !(h)->timing;   /* tapgemm.h: PDL */              \
    ian::coop_finalize_flag() = (h)->coop_finalize;                                                  \
    int _n = (expr);                                                                                 \
    if (_n < 0) return fail(h, IAN_ERR_CUDA, "%s: launch failed: %s", #expr, cudaGetErrorString(cudaGetLastError())); \
    (h)->launches += _n;                                                                             \
  } while (0)

struct Planes {               // NHWC split-plane activation tensor
  __nv_bfloat16* p = nullptr;
  long long plane = 0;
};

struct Plan {
  int n = 0;
  Planes a1, a2, a3, a4, f1, zp, h0, h1, h2, h3, d3, d2, d1, d0;
  float *x = nullptr, *head = nullptr, *z = nullptr, *xhat = nullptr, *gpad = nullptr, *eps = nullptr;
  float* target = nullptr;
  int32_t* boxes = nullptr;
  // full IAN activations (NHWC split planes): block input x, pre-activated t0, mid t2, block output y per scale
  Planes fh0, fx1, ft1, fu1, fy1, fx2, ft2, fu2, fy2, fx3, ft3, fu3, fy3, fh4;
  uint8_t* stroke = nullptr;     // ian_paint_stroke_host staging (allocated on first use)
  float *z0 = nullptr, *ha = nullptr, *rg = nullptr, *tt = nullptr;   // tt: head tap table [n][198][4096]
  // brush backward of the flow models: saved B, head gradient, its im2col operand, and the per-stage gradients
  float *bsave = nullptr, *dpre = nullptr;
  Planes dha2, d4, ds3, du3, dx3, ds2, du2, dx2, ds1, du1, dx1, dfh0;
  // encoder VJP (allocated on the plan's first ian_encode_vjp_* call): gradient planes of the head's pre-BN output, of
  // enc_fc1's and enc_conv4..1's pre-activations; dz staging, dz_iaf, enc_fc1's float32 output gradient, split-K slabs
  bool evjp = false;
  Planes eh, ef1, e4, e3, e2, e1;
  float *edz = nullptr, *edzi = nullptr, *eg = nullptr;
  TapGemm g[L_COUNT];
  TcMaps* maps[L_COUNT] = {nullptr};
  DecOutMaps* decout_maps = nullptr;
  DecOutMaps* conv1_bwd_maps = nullptr;   // encoder VJP: enc_conv1's adjoint on the e1 planes (tensor-core path)
  Conv1OutMap* conv1_out = nullptr;       // TMA-store view of a1 (conv1_tc.cu)
  HeadMaps* head_maps = nullptr;
  // pipelined host API: double-buffered boundary tensors + events (allocated on first use)
  float *sx[2] = {nullptr, nullptr}, *sz[2] = {nullptr, nullptr}, *sxh[2] = {nullptr, nullptr};
  cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr};
  // CUDA graphs of the kernel sequences behind the host entry points (small batches only; see run_graphed)
  struct GraphSlot { cudaGraphExec_t exec = nullptr; int64_t launches = 0; uint64_t key = 0; };
  // decoder parameter VJP (allocated on the plan's first ian_decode_param_vjp_* call): the raw pre-BN sums x of l_dec_fc2 and
  // dec_conv1..3, dL/dh of h0..h3 (before mask and scale), the seed image of dec_out, the weight-gradient descriptors and
  // their split-K slabs, and the partial sums of the small reductions
  bool pvjp = false;
  Planes x0r, x1r, x2r, x3r, dh0, dh1, dh2, dh3;
  float *pseed = nullptr, *pws = nullptr, *ppart = nullptr;
  WgradGemm wg[4];
  WgradMaps* wmaps[4] = {nullptr};
  // decoder JVP (allocated on the plan's first ian_decode_jvp_* call): the tangent of the latent planes, and per decoder
  // forward layer k the tangent of its output (jt[k]) and of its raw pre-BN sum where the forward keeps one (jr[k], IAN.py's
  // block residuals); the tangent sigmoids of the RGB-Beta head, and the head's and dec_out's maps on the tangent planes.
  // The head's tap table tt and ha are reused: the primal head has consumed them when the tangent head runs.
  bool jvp = false;
  Planes jzp, jt[11], jr[11];
  float* jrg = nullptr;
  DecOutMaps* jdecout_maps = nullptr;
  HeadMaps* jhead_maps = nullptr;
  // encoder JVP (allocated on the plan's first ian_encode_jvp_* call): the tangents of a1..a4 and of enc_fc1's output (split
  // planes), enc_fc1's tangent before its activation derivative, the head's tangent [t_mu | t_ls] and t_z_iaf (float32), and
  // the TMA-store view of a1's tangent
  bool ejvp = false;
  Planes jea[4], jef1;
  float *jeg = nullptr, *jeh = nullptr, *jez0 = nullptr;
  Conv1OutMap* jconv1_out = nullptr;
  // latent fit (allocated on the plan's first ian_decode_gauss_newton_* / ian_fit_latent_* call): the normal equations A, g
  // and the Gram's e; per sample the fit's state -- e, lambda, x_hat at z -- and its trial z, x_hat and solve flag; the host
  // form's loss history (grown to the largest iteration count asked for)
  bool gn = false;
  double *gnA = nullptr, *gng = nullptr, *gne = nullptr, *fe = nullptr, *flam = nullptr;
  float *fxh = nullptr, *fxt = nullptr, *fzt = nullptr, *floss = nullptr;
  int* fok = nullptr;
  long long floss_cap = 0;
  // robust fit (allocated on the plan's first ian_robust_gauss_newton_* / ian_fit_latent_robust_* call): the per-sample
  // scale when the caller passes none and asks for none back, and the host form's staging of scale and scale_out
  double* rdl = nullptr;
  // feature fit (allocated on the plan's first ian_feature_gauss_newton_* / ian_fit_latent_features_* call): the target's
  // features g(x) and the current ones g(x_hat), float32 NHWC, layer l's n samples at n * kFeatOff[l] (1.97 MB per image)
  bool feat = false;
  float *ftg = nullptr, *fcur = nullptr;
  // ian_introspect*_host staging: the features, then their tangents, float32 NCHW, laid out as ftg (first host call)
  float* ifeat = nullptr;
  // the features' VJP (allocated on the plan's first ian_introspect_vjp_* call, with the encoder VJP's planes): the
  // cotangents of a1..a3 as split planes NHWC, the res operand of IV_BWD_CONV2..4 (0.92 MB per image)
  bool ivjp = false;
  Planes ivc[3];
  // each batch-statistics stack's tap-GEMM twins: [stack][0] the forward ones (DT_ENC_CONV2..4, DD_DEC_*) on the stack's first
  // call on the plan, [stack][1] the backward-data ones (DT_BWD_*, DD_BWD_*) with their VJP's planes on its first VJP call
  bool bn_twins[2][2] = {};
  enum { G_ENCODE, G_ENCODE_EPS, G_DECODE, G_RECON, G_GRAD, G_EDIT_STEP, G_STROKE, G_VJP, G_ENC_VJP, G_PARAM_VJP, G_JVP, G_ENC_JVP,
         G_ENCODE_PRE, G_FLOW, G_FLOW_VJP, G_FLOW_JVP, G_ENC_PRE_VJP, G_ENC_PRE_JVP, G_COUNT };
  GraphSlot graph[G_COUNT];
  std::vector<void*> allocs;
};

int alloc_planes(ian_handle* h, Plan* pl, Planes& t, long long elems) {
  void* p = nullptr;
  CUDA_TRY(h, cudaMalloc(&p, (size_t)elems * 2 * sizeof(__nv_bfloat16)));
  CUDA_TRY(h, cudaMemsetAsync(p, 0, (size_t)elems * 2 * sizeof(__nv_bfloat16), h->stream));
  pl->allocs.push_back(p);
  t.p = (__nv_bfloat16*)p;
  t.plane = elems;
  return IAN_OK;
}
template <typename T>
int alloc_buf(ian_handle* h, Plan* pl, T*& out, long long elems) {
  void* p = nullptr;
  CUDA_TRY(h, cudaMalloc(&p, (size_t)elems * sizeof(T)));
  CUDA_TRY(h, cudaMemsetAsync(p, 0, (size_t)elems * sizeof(T), h->stream));
  pl->allocs.push_back(p);
  out = (T*)p;
  return IAN_OK;
}

// ---- tap tables --------------------------------------------------------------------------------
// The strided tables are sorted by view.  The tensor-core path runs K chunk-major (tapgemm.h), so the taps of one view run
// back to back on the same 64 channels, and their boxes of that view overlap in all but a one-pixel edge.
void sort_taps_by_view(TapGemm& g) {
  std::stable_sort(g.taps, g.taps + g.phase[0].ntaps, [](const Tap& x, const Tap& y) { return x.view < y.view; });
}
void taps_conv_s2(TapGemm& g) {           // enc_conv: y[p] = sum_i x[2p+i-2] W[i]   (IAN_simple.py:73-116)
  g.nphase = 1;
  g.phase[0] = {0, 25, 0, 0};
  int t = 0;
  for (int i = 0; i < 5; ++i)
    for (int j = 0; j < 5; ++j) {
      const int a = (i - 2) >> 1, r = (i - 2) & 1, b = (j - 2) >> 1, s = (j - 2) & 1;
      g.taps[t++] = {(int16_t)(r * 2 + s), (int16_t)a, (int16_t)b, (int16_t)(i * 5 + j)};
    }
  sort_taps_by_view(g);
  g.sh = g.sw = 2;
  g.osh = g.osw = 1;
}
void taps_deconv_s2(TapGemm& g) {         // dec_conv: y[2p+r] = sum_d x[p+d] W[2+2d-r]   (layers.py:436-483)
  g.nphase = 4;
  int t = 0;
  for (int r = 0; r < 2; ++r)
    for (int s = 0; s < 2; ++s) {
      Phase& ph = g.phase[r * 2 + s];
      ph.tap_begin = t;
      ph.oh0 = r;
      ph.ow0 = s;
      for (int d = (r ? 0 : -1); d <= 1; ++d)
        for (int e = (s ? 0 : -1); e <= 1; ++e) {
          const int ki = 2 + 2 * d - r, kj = 2 + 2 * e - s;
          g.taps[t++] = {0, (int16_t)d, (int16_t)e, (int16_t)(ki * 5 + kj)};
        }
      ph.ntaps = t - ph.tap_begin;
    }
  g.sh = g.sw = 1;
  g.osh = g.osw = 2;
}
void taps_deconv_bwd(TapGemm& g) {        // dx[a] = sum_ki dy[2+2a-ki] W[ki]   (T.grad of the above, API.py:59,64)
  g.nphase = 1;
  g.phase[0] = {0, 25, 0, 0};
  int t = 0;
  for (int ki = 0; ki < 5; ++ki)
    for (int kj = 0; kj < 5; ++kj) {
      const int e = 2 - ki, f = 2 - kj;
      g.taps[t++] = {(int16_t)((e & 1) * 2 + (f & 1)), (int16_t)(e >> 1), (int16_t)(f >> 1), (int16_t)(ki * 5 + kj)};
    }
  sort_taps_by_view(g);
  g.sh = g.sw = 2;
  g.osh = g.osw = 1;
}
void taps_dense(TapGemm& g) {
  g.nphase = 1;
  g.phase[0] = {0, 1, 0, 0};
  g.taps[0] = {0, 0, 0, 0};
  g.sh = g.sw = 1;
  g.osh = g.osw = 1;
}

// distinct tap offsets of an MDC layer (reference layers.py:207-258): 3x3 base, then 3x3 dilated by each s > 0
// (0 in scales = the 1x1 mean filter, which lands on the centre tap).  17 / 25 / 33 offsets for [0,2] / [0,2,3] / [2,3,4].
std::vector<std::pair<int, int>> mdc_offsets(const std::vector<int>& scales) {
  std::vector<std::pair<int, int>> off;
  auto add = [&](int dy, int dx) {
    for (auto& o : off) if (o.first == dy && o.second == dx) return;
    off.push_back({dy, dx});
  };
  for (int i = -1; i <= 1; ++i) for (int j = -1; j <= 1; ++j) add(i, j);
  for (int s : scales) if (s > 0) for (int i = -1; i <= 1; ++i) for (int j = -1; j <= 1; ++j) add(i * s, j * s);
  return off;
}
void taps_mdc(TapGemm& g, const std::vector<int>& scales) {
  const auto off = mdc_offsets(scales);
  g.nphase = 1;
  g.phase[0] = {0, (int)off.size(), 0, 0};
  for (size_t t = 0; t < off.size(); ++t) g.taps[t] = {0, (int16_t)off[t].first, (int16_t)off[t].second, (int16_t)t};
  g.sh = g.sw = 1;
  g.osh = g.osw = 1;
}

void taps_mdc_bwd(TapGemm& g, const std::vector<int>& scales) {   // din[q] = sum_t dout[q - off_t] * comp_t^T
  const auto off = mdc_offsets(scales);
  g.nphase = 1;
  g.phase[0] = {0, (int)off.size(), 0, 0};
  for (size_t t = 0; t < off.size(); ++t) g.taps[t] = {0, (int16_t)(-off[t].first), (int16_t)(-off[t].second), (int16_t)t};
  g.sh = g.sw = 1;
  g.osh = g.osw = 1;
}

void set_io(TapGemm& g, const Planes& a, int n, int Hin, int Win, int Cin, int Hg, int Wg, const DevWeights& w,
            int Hout, int Wout) {
  g.a = a.p; g.a_plane = a.plane;
  g.n_img = n; g.Hin = Hin; g.Win = Win; g.Cin = Cin; g.Hg = Hg; g.Wg = Wg;
  g.b = w.b; g.b_plane = w.plane; g.Cout = w.Cout;
  g.scale = w.scale; g.shift = w.shift; g.scale_pix_stride = 0;
  g.Hout = Hout; g.Wout = Wout;
  g.ksplit = 1; g.ws = nullptr; g.mask = nullptr; g.out = nullptr; g.out_f32 = nullptr; g.out_plane = 0;
  g.res = nullptr; g.res_plane = 0; g.out_raw = nullptr; g.out_raw_plane = 0; g.out_f32_t = nullptr; g.cout_real = 0;
}

int choose_ksplit(const TapGemm& g) {
  // fill ~one wave of the SMs when the output tile count is small; keep >= 4 K steps per CTA
  const int bn = (g.Cout % 128 == 0) ? 128 : 16;   // the tile width tc_build_maps picks
  const int M = g.n_img * g.Hg * g.Wg;
  const int ctas = ((M + 127) / 128) * (g.Cout / bn) * g.nphase;
  int min_it = 1 << 30;
  for (int p = 0; p < g.nphase; ++p) {
    const int it = g.phase[p].ntaps * (g.Cin / 64);
    if (it < min_it) min_it = it;
  }
  int ks = tc_num_sms() / ctas;
  if (ks > min_it / 4) ks = min_it / 4;
  if (ks < 1) ks = 1;
  if (ks > 64) ks = 64;
  return ks;
}

// A fixed sequence of tap-GEMM layers, in run order
struct LayerList {
  int n = 0;
  int l[32] = {};
  const int* begin() const { return l; }
  const int* end() const { return l + n; }
  LayerList operator+(const LayerList& o) const {
    LayerList r = *this;
    for (int x : o) r.l[r.n++] = x;
    return r;
  }
};

// The tap-GEMM layers of each graph, read by the run functions and by finish_maps.  The encoder (IAN_simple.py:84-126;
// its enc_fc1 activation differs per graph, not its layers) and the encoder VJP are shared by all three graphs.
const LayerList kEncoder = {5, {L_ENC_CONV2, L_ENC_CONV3, L_ENC_CONV4, L_ENC_FC1, L_ENC_HEAD}};
const LayerList kEncoderBwd = {5, {E_BWD_HEAD, E_BWD_FC1, E_BWD_CONV4, E_BWD_CONV3, E_BWD_CONV2}};
// the encoder's tangent (JVP) chain: kEncoderJvp.l[k] is the tangent twin of kEncoder.l[k]
const LayerList kEncoderJvp = {5, {JE_ENC_CONV2, JE_ENC_CONV3, JE_ENC_CONV4, JE_ENC_FC1, JE_ENC_HEAD}};
// the decoder forward, its backward-data from the last layer down to z, and its tangent (JVP) chain: jvp[k] = jvp_twin(fwd[k])
struct DecoderLayers { LayerList fwd, bwd, jvp; };
const DecoderLayers kSimpleDecoder = {{4, {L_DEC_FC2, L_DEC_CONV1, L_DEC_CONV2, L_DEC_CONV3}},
                                      {4, {L_BWD_CONV3, L_BWD_CONV2, L_BWD_CONV1, L_BWD_FC2}},
                                      {4, {J_DEC_FC2, J_DEC_CONV1, J_DEC_CONV2, J_DEC_CONV3}}};
const DecoderLayers kV1Decoder = {{5, {L_DEC_FC2, L_DEC_CONV1, L_DEC_CONV2, L_DEC_CONV3, F_DEC_CONV4}},
                                  {6, {F_BWD_HEAD, F_BWD_CONV4, L_BWD_CONV3, L_BWD_CONV2, L_BWD_CONV1, L_BWD_FC2}},
                                  {5, {J_DEC_FC2, J_DEC_CONV1, J_DEC_CONV2, J_DEC_CONV3, JF_DEC_CONV4}}};
const DecoderLayers kFullDecoder = {{11, {F_DEC_FC2, F_DEC_CONV1, F_MD1A, F_MD1B, F_DEC_CONV2, F_MD2A, F_MD2B, F_DEC_CONV3,
                                          F_MD3A, F_MD3B, F_DEC_CONV4}},
                                    {12, {F_BWD_HEAD, F_BWD_CONV4, F_BWD_MD3B, F_BWD_MD3A, F_BWD_CONV3, F_BWD_MD2B,
                                          F_BWD_MD2A, F_BWD_CONV2, F_BWD_MD1B, F_BWD_MD1A, F_BWD_CONV1, F_BWD_FC2}},
                                    {11, {JF_DEC_FC2, JF_DEC_CONV1, JF_MD1A, JF_MD1B, JF_DEC_CONV2, JF_MD2A, JF_MD2B, JF_DEC_CONV3,
                                          JF_MD3A, JF_MD3B, JF_DEC_CONV4}}};
const DecoderLayers& decoder_layers(const ian_handle* h) {
  return h->model_kind == IAN_MODEL_FULL ? kFullDecoder : h->model_kind == IAN_MODEL_V1 ? kV1Decoder : kSimpleDecoder;
}

// Tensor maps of `layers`, their split-K factors, and one split-K workspace shared by them (they run back to back on one
// stream): [ksplit][pixel][Cout] float32 slabs, sized for the largest user.
// Small batches (NPE runs batch 1): a layer with fewer tiles than SMs would stream its weights through a handful of
// SMs.  Every such layer is marked (ksplit = 0: "choose") so choose_ksplit() can spread K over the chip.
int finish_maps(ian_handle* h, Plan* pl, const LayerList& layers) {
  long long need = 0;
  for (int l : layers) {
    TapGemm& g = pl->g[l];
    const int bn = (g.Cout % 256 == 0) ? 256 : (g.Cout % 128 == 0) ? 128 : 16;
    const long long tiles = (long long)((g.n_img * g.Hg * g.Wg + 127) / 128) * (g.Cout / bn) * g.nphase;
    if (!g.out_f32_t && tiles <= 74) g.ksplit = 0;
    char err[256] = {0};
    pl->maps[l] = tc_build_maps(g, err, sizeof(err));
    if (!pl->maps[l]) return fail(h, IAN_ERR_CUDA, "layer %s: %s", kLayerNames[l], err);
    if (g.ksplit == 0) g.ksplit = h->splitk ? choose_ksplit(g) : 1;
    if (g.ksplit > 1) {
      g.ws_slab = (long long)g.n_img * g.Hout * g.Wout * g.Cout;
      need = std::max(need, g.ws_slab * g.ksplit);
    }
  }
  if (need == 0) return IAN_OK;
  float* ws = nullptr;
  int rc = alloc_buf(h, pl, ws, need);
  if (rc != IAN_OK) return rc;
  for (int l : layers)
    if (pl->g[l].ksplit > 1) pl->g[l].ws = ws;
  return IAN_OK;
}

// decoder of IANv1 (reference IANv1.py:125-201): dense (linear) -> 4 x [deconv, BN, relu] -> RGB-Beta head.  The last deconv
// has 64 output channels; it is stored 128 wide (upper half zero weights) so the head GEMM keeps Cin % 64 == 0 tiles.
void wire_decoder_v1(ian_handle* h, Plan* pl) {
  TapGemm* g = pl->g;
  const int n = pl->n;
  auto outp = [](TapGemm& gg, const Planes& t) { gg.out = t.p; gg.out_plane = t.plane; };
  set_io(g[L_DEC_FC2], pl->zp, n, 1, 1, 128, 1, 1, h->w[L_DEC_FC2], 1, 1); taps_dense(g[L_DEC_FC2]);
  g[L_DEC_FC2].act = ACT_NONE; outp(g[L_DEC_FC2], pl->h0);
  set_io(g[L_DEC_CONV1], pl->h0, n, 4, 4, 1024, 4, 4, h->w[L_DEC_CONV1], 8, 8); taps_deconv_s2(g[L_DEC_CONV1]);
  g[L_DEC_CONV1].act = ACT_RELU; outp(g[L_DEC_CONV1], pl->h1);
  set_io(g[L_DEC_CONV2], pl->h1, n, 8, 8, 512, 8, 8, h->w[L_DEC_CONV2], 16, 16); taps_deconv_s2(g[L_DEC_CONV2]);
  g[L_DEC_CONV2].act = ACT_RELU; outp(g[L_DEC_CONV2], pl->h2);
  set_io(g[L_DEC_CONV3], pl->h2, n, 16, 16, 256, 16, 16, h->w[L_DEC_CONV3], 32, 32); taps_deconv_s2(g[L_DEC_CONV3]);
  g[L_DEC_CONV3].act = ACT_RELU; outp(g[L_DEC_CONV3], pl->h3);
  set_io(g[F_DEC_CONV4], pl->h3, n, 32, 32, 128, 32, 32, h->w[F_DEC_CONV4], 64, 64); taps_deconv_s2(g[F_DEC_CONV4]);
  g[F_DEC_CONV4].act = ACT_RELU; outp(g[F_DEC_CONV4], pl->fh4);
  set_io(g[F_HEAD], pl->fh4, n, 64, 64, 128, 64, 64, h->w[F_HEAD], 64, 64); taps_dense(g[F_HEAD]);
  g[F_HEAD].act = ACT_NONE; g[F_HEAD].out_f32_t = pl->tt; g[F_HEAD].cout_real = 198;
  // ---- brush backward (T.grad of API.py:59,64 on this graph): head GEMM, then the four deconvs' backward-data and the dense
  auto bwd = [&](int l, const Planes& in, int Hin, int Cin, const Planes& out, const Planes* mask, int act) {
    set_io(g[l], in, n, Hin, Hin, Cin, Hin / 2, Hin / 2, h->w[l], Hin / 2, Hin / 2); taps_deconv_bwd(g[l]);
    g[l].act = act; g[l].mask = mask ? mask->p : nullptr; g[l].mask_slope = 0.f; outp(g[l], out);
  };
  set_io(g[F_BWD_HEAD], pl->dha2, n, 64, 64, 256, 64, 64, h->w[F_BWD_HEAD], 64, 64); taps_dense(g[F_BWD_HEAD]);
  g[F_BWD_HEAD].act = ACT_MASK; g[F_BWD_HEAD].mask = pl->fh4.p; outp(g[F_BWD_HEAD], pl->d4);
  bwd(F_BWD_CONV4, pl->d4, 64, 128, pl->d3, &pl->h3, ACT_MASK);
  bwd(L_BWD_CONV3, pl->d3, 32, 128, pl->d2, &pl->h2, ACT_MASK);
  bwd(L_BWD_CONV2, pl->d2, 16, 256, pl->d1, &pl->h1, ACT_MASK);
  bwd(L_BWD_CONV1, pl->d1, 8, 512, pl->d0, nullptr, ACT_NONE);          // l_dec_fc2 is linear here (IANv1.py:125-130)
  set_io(g[L_BWD_FC2], pl->d0, n, 1, 1, 16384, 1, 1, h->w[L_BWD_FC2], 1, 1); taps_dense(g[L_BWD_FC2]);
  g[L_BWD_FC2].act = ACT_NONE; g[L_BWD_FC2].out_f32 = pl->gpad; g[L_BWD_FC2].ksplit = 0;
}

// decoder of the full IAN (reference IAN.py:129-207): dense -> 3 x (deconv, MDBLOCK) -> deconv -> RGB-Beta head
void wire_decoder_full(ian_handle* h, Plan* pl) {
  TapGemm* g = pl->g;
  const int n = pl->n;
  auto outp = [](TapGemm& gg, const Planes& t) { gg.out = t.p; gg.out_plane = t.plane; };
  set_io(g[F_DEC_FC2], pl->zp, n, 1, 1, 128, 1, 1, h->w[F_DEC_FC2], 1, 1); taps_dense(g[F_DEC_FC2]);
  g[F_DEC_FC2].act = ACT_LRELU; outp(g[F_DEC_FC2], pl->fh0);
  struct Stage { int dconv, mda, mdb; const Planes *in, *x, *t, *u, *y; int Hin, Cin, Cout; std::vector<int> scales; };
  const Stage st[3] = {{F_DEC_CONV1, F_MD1A, F_MD1B, &pl->fh0, &pl->fx1, &pl->ft1, &pl->fu1, &pl->fy1, 4, 512, 512, {0, 2}},
                       {F_DEC_CONV2, F_MD2A, F_MD2B, &pl->fy1, &pl->fx2, &pl->ft2, &pl->fu2, &pl->fy2, 8, 512, 256, {0, 2, 3}},
                       {F_DEC_CONV3, F_MD3A, F_MD3B, &pl->fy2, &pl->fx3, &pl->ft3, &pl->fu3, &pl->fy3, 16, 256, 128, {0, 2, 3}}};
  for (const Stage& s : st) {
    const int Ho = 2 * s.Hin;
    // deconv: raw sum -> x (block residual), lrelu(BN0(x)) -> t    (layers.py:413: BN(incoming) strips the bias)
    set_io(g[s.dconv], *s.in, n, s.Hin, s.Hin, s.Cin, s.Hin, s.Hin, h->w[s.dconv], Ho, Ho); taps_deconv_s2(g[s.dconv]);
    g[s.dconv].act = ACT_LRELU; outp(g[s.dconv], *s.t);
    g[s.dconv].out_raw = s.x->p; g[s.dconv].out_raw_plane = s.x->plane;
    // MDCL 1: lrelu(BN1(.)) ; MDCL 2: lrelu(BN2(x + .))
    set_io(g[s.mda], *s.t, n, Ho, Ho, s.Cout, Ho, Ho, h->w[s.mda], Ho, Ho); taps_mdc(g[s.mda], s.scales);
    g[s.mda].act = ACT_LRELU; outp(g[s.mda], *s.u);
    set_io(g[s.mdb], *s.u, n, Ho, Ho, s.Cout, Ho, Ho, h->w[s.mdb], Ho, Ho); taps_mdc(g[s.mdb], s.scales);
    g[s.mdb].act = ACT_LRELU; outp(g[s.mdb], *s.y);
    g[s.mdb].res = s.x->p; g[s.mdb].res_plane = s.x->plane;
  }
  set_io(g[F_DEC_CONV4], pl->fy3, n, 32, 32, 128, 32, 32, h->w[F_DEC_CONV4], 64, 64); taps_deconv_s2(g[F_DEC_CONV4]);
  g[F_DEC_CONV4].act = ACT_LRELU; outp(g[F_DEC_CONV4], pl->fh4);
  // RGB-Beta head: ONE dense 128 -> 33 taps x 6 filters GEMM (no shifts: the feature map is staged once, not 33
  // times), written channel-major; the dilated taps are applied afterwards as coalesced shifted reads (head_gather)
  set_io(g[F_HEAD], pl->fh4, n, 64, 64, 128, 64, 64, h->w[F_HEAD], 64, 64); taps_dense(g[F_HEAD]);
  g[F_HEAD].act = ACT_NONE; g[F_HEAD].out_f32_t = pl->tt; g[F_HEAD].cout_real = 198;
  // ---- brush backward (T.grad of API.py:59,64 on this graph).  LeakyRectify(0.2) backward = mask slope 0.2 on the sign of
  // the stored forward activation; MDBLOCK (layers.py:411-416) y = lrelu(BN2(x + M2(u))), u = lrelu(BN1(M1(t))), t = lrelu(BN0(x)):
  //   ds = dy * lrelu'(y) * s2 ;  du = M2^T(ds) * lrelu'(u) * s1 ;  dx = M1^T(du) * lrelu'(t) * s0 + ds
  set_io(g[F_BWD_HEAD], pl->dha2, n, 64, 64, 256, 64, 64, h->w[F_BWD_HEAD], 64, 64); taps_dense(g[F_BWD_HEAD]);
  g[F_BWD_HEAD].act = ACT_MASK; g[F_BWD_HEAD].mask = pl->fh4.p; g[F_BWD_HEAD].mask_slope = 0.2f; outp(g[F_BWD_HEAD], pl->d4);
  struct BStage { int dconv, mdb, mda; const Planes *din, *ds, *du, *dx, *y, *u, *t; int Hin, Cin, Cout; std::vector<int> scales; };
  // dconv: backward-data of the deconv ABOVE the block (its input gradient `din` lives at 2x the block's resolution)
  const BStage bs[3] = {{F_BWD_CONV4, F_BWD_MD3B, F_BWD_MD3A, &pl->d4, &pl->ds3, &pl->du3, &pl->dx3, &pl->fy3, &pl->fu3, &pl->ft3, 64, 128, 128, {0, 2, 3}},
                        {F_BWD_CONV3, F_BWD_MD2B, F_BWD_MD2A, &pl->dx3, &pl->ds2, &pl->du2, &pl->dx2, &pl->fy2, &pl->fu2, &pl->ft2, 32, 128, 256, {0, 2, 3}},
                        {F_BWD_CONV2, F_BWD_MD1B, F_BWD_MD1A, &pl->dx2, &pl->ds1, &pl->du1, &pl->dx1, &pl->fy1, &pl->fu1, &pl->ft1, 16, 256, 512, {0, 2}}};
  for (const BStage& b : bs) {
    const int Ho = b.Hin / 2;
    set_io(g[b.dconv], *b.din, n, b.Hin, b.Hin, b.Cin, Ho, Ho, h->w[b.dconv], Ho, Ho); taps_deconv_bwd(g[b.dconv]);
    g[b.dconv].act = ACT_MASK; g[b.dconv].mask = b.y->p; g[b.dconv].mask_slope = 0.2f; outp(g[b.dconv], *b.ds);
    set_io(g[b.mdb], *b.ds, n, Ho, Ho, b.Cout, Ho, Ho, h->w[b.mdb], Ho, Ho); taps_mdc_bwd(g[b.mdb], b.scales);
    g[b.mdb].act = ACT_MASK; g[b.mdb].mask = b.u->p; g[b.mdb].mask_slope = 0.2f; outp(g[b.mdb], *b.du);
    set_io(g[b.mda], *b.du, n, Ho, Ho, b.Cout, Ho, Ho, h->w[b.mda], Ho, Ho); taps_mdc_bwd(g[b.mda], b.scales);
    g[b.mda].act = ACT_MASK; g[b.mda].mask = b.t->p; g[b.mda].mask_slope = 0.2f; outp(g[b.mda], *b.dx);
    g[b.mda].res = b.ds->p; g[b.mda].res_plane = b.ds->plane; g[b.mda].res_after = 1;
  }
  set_io(g[F_BWD_CONV1], pl->dx1, n, 8, 8, 512, 4, 4, h->w[F_BWD_CONV1], 4, 4); taps_deconv_bwd(g[F_BWD_CONV1]);
  g[F_BWD_CONV1].act = ACT_MASK; g[F_BWD_CONV1].mask = pl->fh0.p; g[F_BWD_CONV1].mask_slope = 0.2f; outp(g[F_BWD_CONV1], pl->dfh0);
  set_io(g[F_BWD_FC2], pl->dfh0, n, 1, 1, 8192, 1, 1, h->w[F_BWD_FC2], 1, 1); taps_dense(g[F_BWD_FC2]);
  g[F_BWD_FC2].act = ACT_NONE; g[F_BWD_FC2].out_f32 = pl->gpad; g[F_BWD_FC2].ksplit = 0;
}

// decoder of IAN_simple (IAN_simple.py:129-170) and its backward-data for the latent brush (T.grad at API.py:59,64)
void wire_decoder_simple(ian_handle* h, Plan* pl) {
  TapGemm* g = pl->g;
  const int n = pl->n;
  set_io(g[L_DEC_FC2], pl->zp, n, 1, 1, 128, 1, 1, h->w[L_DEC_FC2], 1, 1); taps_dense(g[L_DEC_FC2]);
  g[L_DEC_FC2].act = ACT_RELU; g[L_DEC_FC2].out = pl->h0.p; g[L_DEC_FC2].out_plane = pl->h0.plane;
  set_io(g[L_DEC_CONV1], pl->h0, n, 4, 4, 1024, 4, 4, h->w[L_DEC_CONV1], 8, 8); taps_deconv_s2(g[L_DEC_CONV1]);
  g[L_DEC_CONV1].act = ACT_RELU; g[L_DEC_CONV1].out = pl->h1.p; g[L_DEC_CONV1].out_plane = pl->h1.plane;
  set_io(g[L_DEC_CONV2], pl->h1, n, 8, 8, 512, 8, 8, h->w[L_DEC_CONV2], 16, 16); taps_deconv_s2(g[L_DEC_CONV2]);
  g[L_DEC_CONV2].act = ACT_RELU; g[L_DEC_CONV2].out = pl->h2.p; g[L_DEC_CONV2].out_plane = pl->h2.plane;
  set_io(g[L_DEC_CONV3], pl->h2, n, 16, 16, 256, 16, 16, h->w[L_DEC_CONV3], 32, 32); taps_deconv_s2(g[L_DEC_CONV3]);
  g[L_DEC_CONV3].act = ACT_RELU; g[L_DEC_CONV3].out = pl->h3.p; g[L_DEC_CONV3].out_plane = pl->h3.plane;
  set_io(g[L_BWD_CONV3], pl->d3, n, 32, 32, 128, 16, 16, h->w[L_BWD_CONV3], 16, 16); taps_deconv_bwd(g[L_BWD_CONV3]);
  g[L_BWD_CONV3].act = ACT_MASK; g[L_BWD_CONV3].mask = pl->h2.p; g[L_BWD_CONV3].out = pl->d2.p; g[L_BWD_CONV3].out_plane = pl->d2.plane;
  set_io(g[L_BWD_CONV2], pl->d2, n, 16, 16, 256, 8, 8, h->w[L_BWD_CONV2], 8, 8); taps_deconv_bwd(g[L_BWD_CONV2]);
  g[L_BWD_CONV2].act = ACT_MASK; g[L_BWD_CONV2].mask = pl->h1.p; g[L_BWD_CONV2].out = pl->d1.p; g[L_BWD_CONV2].out_plane = pl->d1.plane;
  set_io(g[L_BWD_CONV1], pl->d1, n, 8, 8, 512, 4, 4, h->w[L_BWD_CONV1], 4, 4); taps_deconv_bwd(g[L_BWD_CONV1]);
  g[L_BWD_CONV1].act = ACT_MASK; g[L_BWD_CONV1].mask = pl->h0.p; g[L_BWD_CONV1].out = pl->d0.p; g[L_BWD_CONV1].out_plane = pl->d0.plane;
  g[L_BWD_CONV1].scale_pix_stride = 1024;   // bnorm_dec_fc2 is per FEATURE (pixel, channel)
  set_io(g[L_BWD_FC2], pl->d0, n, 1, 1, 16384, 1, 1, h->w[L_BWD_FC2], 1, 1); taps_dense(g[L_BWD_FC2]);
  g[L_BWD_FC2].act = ACT_NONE; g[L_BWD_FC2].out_f32 = pl->gpad; g[L_BWD_FC2].ksplit = 0;
}

int build_plan(ian_handle* h, int n, Plan** out) {
  Plan* pl = new Plan();
  pl->n = n;
  const long long N = n;
  int rc;
#define AP(t, e) if ((rc = alloc_planes(h, pl, pl->t, (e))) != IAN_OK) return rc;
#define AB(t, e) if ((rc = alloc_buf(h, pl, pl->t, (e))) != IAN_OK) return rc;
  const bool full = h->model_kind == IAN_MODEL_FULL, v1 = h->model_kind == IAN_MODEL_V1;
  AP(a1, N * 32 * 32 * 128) AP(a2, N * 16 * 16 * 256) AP(a3, N * 8 * 8 * 512) AP(a4, N * 4 * 4 * 1024)
  AP(f1, N * 1024) AP(zp, N * 128)
  AB(x, N * 3 * 4096) AB(head, N * 256) AB(z, N * 100) AB(xhat, N * 3 * 4096) AB(eps, N * 100)
  if (!full) {
    AP(h0, N * 16384) AP(h1, N * 8 * 8 * 512) AP(h2, N * 16 * 16 * 256) AP(h3, N * 32 * 32 * 128)
  }
  if (v1) {
    AP(fh4, N * 4096 * 128)
    AB(z0, N * 100) AB(ha, N * 4096 * 16) AB(rg, N * 4096 * 4) AB(tt, N * 198 * 4096)
    AB(bsave, N * 4096 * 2) AB(dpre, N * 4096 * 8) AP(dha2, N * 4096 * 256) AP(d4, N * 4096 * 128)
    AP(d3, N * 32 * 32 * 128) AP(d2, N * 16 * 16 * 256) AP(d1, N * 8 * 8 * 512) AP(d0, N * 16384)
    AB(gpad, N * 128) AB(target, N * 3 * 4096) AB(boxes, N * 4)
  } else if (!full) {
    AP(d3, N * 32 * 32 * 128) AP(d2, N * 16 * 16 * 256) AP(d1, N * 8 * 8 * 512) AP(d0, N * 16384)
    AB(gpad, N * 128) AB(target, N * 3 * 4096) AB(boxes, N * 4)
  } else {
    AP(fh0, N * 8192)
    AP(fx1, N * 64 * 512) AP(ft1, N * 64 * 512) AP(fu1, N * 64 * 512) AP(fy1, N * 64 * 512)
    AP(fx2, N * 256 * 256) AP(ft2, N * 256 * 256) AP(fu2, N * 256 * 256) AP(fy2, N * 256 * 256)
    AP(fx3, N * 1024 * 128) AP(ft3, N * 1024 * 128) AP(fu3, N * 1024 * 128) AP(fy3, N * 1024 * 128)
    AP(fh4, N * 4096 * 128)
    AB(z0, N * 100) AB(ha, N * 4096 * 16) AB(rg, N * 4096 * 4) AB(tt, N * 198 * 4096)
    AB(bsave, N * 4096 * 2) AB(dpre, N * 4096 * 8) AP(dha2, N * 4096 * 256) AP(d4, N * 4096 * 128)
    AP(ds3, N * 1024 * 128) AP(du3, N * 1024 * 128) AP(dx3, N * 1024 * 128)
    AP(ds2, N * 256 * 256) AP(du2, N * 256 * 256) AP(dx2, N * 256 * 256)
    AP(ds1, N * 64 * 512) AP(du1, N * 64 * 512) AP(dx1, N * 64 * 512)
    AP(dfh0, N * 8192)
    AB(gpad, N * 128) AB(target, N * 3 * 4096) AB(boxes, N * 4)
  }
#undef AP
#undef AB

  TapGemm* g = pl->g;
  memset(g, 0, sizeof(TapGemm) * L_COUNT);
  // ---- encoder (IAN_simple.py:84-126)
  set_io(g[L_ENC_CONV2], pl->a1, n, 32, 32, 128, 16, 16, h->w[L_ENC_CONV2], 16, 16); taps_conv_s2(g[L_ENC_CONV2]);
  g[L_ENC_CONV2].act = ACT_LRELU; g[L_ENC_CONV2].out = pl->a2.p; g[L_ENC_CONV2].out_plane = pl->a2.plane;
  set_io(g[L_ENC_CONV3], pl->a2, n, 16, 16, 256, 8, 8, h->w[L_ENC_CONV3], 8, 8); taps_conv_s2(g[L_ENC_CONV3]);
  g[L_ENC_CONV3].act = ACT_LRELU; g[L_ENC_CONV3].out = pl->a3.p; g[L_ENC_CONV3].out_plane = pl->a3.plane;
  set_io(g[L_ENC_CONV4], pl->a3, n, 8, 8, 512, 4, 4, h->w[L_ENC_CONV4], 4, 4); taps_conv_s2(g[L_ENC_CONV4]);
  g[L_ENC_CONV4].act = ACT_LRELU; g[L_ENC_CONV4].out = pl->a4.p; g[L_ENC_CONV4].out_plane = pl->a4.plane;
  set_io(g[L_ENC_FC1], pl->a4, n, 1, 1, 16384, 1, 1, h->w[L_ENC_FC1], 1, 1); taps_dense(g[L_ENC_FC1]);
  g[L_ENC_FC1].act = has_flow(h) ? ACT_RELU : ACT_ELU;   // IAN.py:118 / IANv1.py:109 use rectify, IAN_simple.py:121 elu
  g[L_ENC_FC1].out = pl->f1.p; g[L_ENC_FC1].out_plane = pl->f1.plane; g[L_ENC_FC1].ksplit = 0;
  set_io(g[L_ENC_HEAD], pl->f1, n, 1, 1, 1024, 1, 1, h->w[L_ENC_HEAD], 1, 1); taps_dense(g[L_ENC_HEAD]);
  g[L_ENC_HEAD].act = ACT_NONE; g[L_ENC_HEAD].out_f32 = pl->head;
  {                                                       // (both paths: ian_set_path may switch a live handle)
    char err[256] = {0};
    pl->conv1_out = conv1_build_out_map(pl->a1.p, pl->a1.plane, n, err, sizeof(err));
    if (!pl->conv1_out) return fail(h, IAN_ERR_CUDA, "enc_conv1: %s", err);
  }
  if (full) wire_decoder_full(h, pl);
  else if (v1) wire_decoder_v1(h, pl);
  else wire_decoder_simple(h, pl);
  const DecoderLayers& dec = decoder_layers(h);
  const LayerList head = {has_flow(h) ? 1 : 0, {F_HEAD}};   // the head GEMM of the verification path (run_head)
  if ((rc = finish_maps(h, pl, kEncoder + dec.fwd + head + dec.bwd)) != IAN_OK) return rc;
  char err[256] = {0};
  if (has_flow(h)) {
    pl->head_maps = head_build_maps(pl->fh4.p, pl->fh4.plane, n, h->head_tc_wt, 3 * 80 * 128, err, sizeof(err));
    if (!pl->head_maps) return fail(h, IAN_ERR_CUDA, "rgb head: %s", err);
  } else {
    pl->decout_maps = decout_build_maps(pl->h3.p, pl->h3.plane, n, h->decout_tc_wt, 80 * 128, err, sizeof(err));
    if (!pl->decout_maps) return fail(h, IAN_ERR_CUDA, "dec_out: %s", err);
  }
  *out = pl;
  return IAN_OK;
}

void free_plan(Plan* pl) {
  for (void* p : pl->allocs) cudaFree(p);
  for (int s = 0; s < 2; ++s) {
    if (pl->ev_h2d[s]) cudaEventDestroy(pl->ev_h2d[s]);
    if (pl->ev_comp[s]) cudaEventDestroy(pl->ev_comp[s]);
    if (pl->ev_d2h[s]) cudaEventDestroy(pl->ev_d2h[s]);
  }
  for (int l = 0; l < L_COUNT; ++l) if (pl->maps[l]) tc_free_maps(pl->maps[l]);
  for (auto* m : pl->wmaps) if (m) wgrad_free_maps(m);
  if (pl->decout_maps) decout_free_maps(pl->decout_maps);
  if (pl->conv1_bwd_maps) decout_free_maps(pl->conv1_bwd_maps);
  if (pl->conv1_out) conv1_free_out_map(pl->conv1_out);
  if (pl->head_maps) head_free_maps(pl->head_maps);
  if (pl->jdecout_maps) decout_free_maps(pl->jdecout_maps);
  if (pl->jhead_maps) head_free_maps(pl->jhead_maps);
  if (pl->jconv1_out) conv1_free_out_map(pl->jconv1_out);
  cudaFree(pl->floss);
  for (auto& gs : pl->graph) if (gs.exec) cudaGraphExecDestroy(gs.exec);
  delete pl;
}

int get_plan(ian_handle* h, int n, Plan** out) {
  auto it = h->plans.find(n);
  if (it != h->plans.end()) { *out = it->second; return IAN_OK; }
  Plan* pl = nullptr;
  int rc = build_plan(h, n, &pl);
  if (rc != IAN_OK) { if (pl) free_plan(pl); return rc; }
  h->plans[n] = pl;
  *out = pl;
  return IAN_OK;
}

// ---- one tap-GEMM layer -------------------------------------------------------------------------
// CUDA-event pair around one kernel when layer timing is on
struct ScopedTimer {
  ian_handle* h; int slot; cudaStream_t st; ian_handle::Timed tm{}; bool on;
  ScopedTimer(ian_handle* h_, int slot_, cudaStream_t st_) : h(h_), slot(slot_), st(st_), on(h_->timing) {
    if (on) { cudaEventCreate(&tm.e0); cudaEventCreate(&tm.e1); cudaEventRecord(tm.e0, st); }
  }
  ~ScopedTimer() {
    if (on) { cudaEventRecord(tm.e1, st); h->timed[slot].push_back(tm); }
  }
};

// Host calls on plans of at most kGraphMaxBatch samples replay a captured CUDA graph (run_graphed).
constexpr int kGraphMaxBatch = 32;

int run_gemm(ian_handle* h, Plan* pl, int l, cudaStream_t st) {
  TapGemm g = pl->g[l];
  if (g.ksplit < 1) return fail(h, IAN_ERR_INVALID, "layer %s is not part of this plan", kLayerNames[l]);
  g.passes = h->passes;
  g.out_t_bf16 = (g.out_f32_t && h->passes == 1) ? 1 : 0;   // bf16 mode: the head's tap table travels as bf16
  // The stream-K epoch is a kernel argument, so a captured graph cannot replay stream-K.  A plan small enough to be
  // captured therefore runs whole tiles on every launch form (graph, plain launches, device-pointer calls) unless
  // stream-K is forced, so all of them compute the same bits.
  const bool sk_ok = !h->capturing && (h->streamk == 2 || pl->n > kGraphMaxBatch);
  g.sk_ws = (h->streamk && sk_ok) ? h->sk_ws : nullptr;
  g.sk_force = h->streamk == 2 ? 1 : 0;
  g.sk_flags = h->sk_flags;
  g.sk_epoch = ++h->sk_epoch;
  g.epi_tma = h->epi_tma ? 1 : 0;
  ian_handle::Timed tm{};
  if (h->timing) {
    CUDA_TRY(h, cudaEventCreate(&tm.e0));
    CUDA_TRY(h, cudaEventCreate(&tm.e1));
  }
  if (h->path == IAN_PATH_SIMT) {
    g.ksplit = 1;
    g.ws = nullptr;
    if (h->timing) CUDA_TRY(h, cudaEventRecord(tm.e0, st));
    LAUNCH_TRY(h, launch_tapgemm_simt(g, st));
    if (h->timing) CUDA_TRY(h, cudaEventRecord(tm.e1, st));
  } else {
    if (h->timing) CUDA_TRY(h, cudaEventRecord(tm.e0, st));
    LAUNCH_TRY(h, launch_tapgemm_tc(g, pl->maps[l], st));
    if (h->timing) CUDA_TRY(h, cudaEventRecord(tm.e1, st));
    if (g.ksplit > 1) LAUNCH_TRY(h, launch_splitk_finalize(g, st));
  }
  if (h->timing) h->timed[l].push_back(tm);
  return IAN_OK;
}

// z_pre (nullable): the pre-flow latent l_Z_IAF (= z itself for IAN_simple)
int run_encode(ian_handle* h, Plan* pl, const float* x, const float* eps, float* z, cudaStream_t st, float* z_pre = nullptr) {
  const int n = pl->n;
  {
    ScopedTimer tm(h, T_CONV1, st);
    if (h->path == IAN_PATH_TC)
      LAUNCH_TRY(h, launch_conv1_tc(h->conv1_maps, pl->conv1_out, x, h->conv1_b, n, st));
    else
      LAUNCH_TRY(h, launch_conv1(x, h->conv1_wt, h->conv1_b, pl->a1.p, pl->a1.plane, n, st));
  }
  int rc;
  for (int l : kEncoder)
    if ((rc = run_gemm(h, pl, l, st)) != IAN_OK) return rc;
  if (has_flow(h)) {
    // l_Z_IAF = mu (+ exp(ls) eps), then l_Z = IAF(l_Z_IAF; MADE_mu, MADE_ls)   (IAN.py:126-128)
    LAUNCH_TRY(h, launch_sample(pl->head, eps, z_pre ? z_pre : pl->z0, nullptr, 0, n, st));
    LAUNCH_TRY(h, launch_made_iaf(z_pre ? z_pre : pl->z0, h->made_w, h->made_b, z, pl->zp.p, pl->zp.plane, n, st));
    return IAN_OK;
  }
  LAUNCH_TRY(h, launch_sample(pl->head, eps, z, pl->zp.p, pl->zp.plane, n, st));
  if (z_pre) CUDA_TRY(h, cudaMemcpyAsync(z_pre, z, (size_t)n * 400, cudaMemcpyDeviceToDevice, st));
  return IAN_OK;
}

// RGB-Beta head (IAN.py:183-207) from the feature map fh4.  Tensor-core path: head_tc.cu (dense GEMM + on-chip tap gather,
// then the autoregressive part in one kernel).  Verification path: the dense GEMM into the HBM tap table + gather + the
// three per-pixel kernels of round 1 -- a second, independent formulation.
int run_head(ian_handle* h, Plan* pl, float* xhat, cudaStream_t st) {
  if (h->path == IAN_PATH_TC) {
    {
      ScopedTimer tm(h, F_HEAD, st);
      LAUNCH_TRY(h, launch_head_tc(pl->head_maps, h->passes, pl->ha, pl->n, st));
    }
    LAUNCH_TRY(h, launch_rgb_beta_head(pl->ha, 1, pl->rg, h->head_taps, h->head_wgb, h->head_wbb, h->head_ntaps, xhat, pl->bsave, pl->n, st));
    return IAN_OK;
  }
  int rc;
  if ((rc = run_gemm(h, pl, F_HEAD, st)) != IAN_OK) return rc;
  LAUNCH_TRY(h, launch_head_gather(pl->tt, h->passes == 1 ? 1 : 0, h->head_taps, h->head_ntaps, pl->ha, pl->n, st));
  LAUNCH_TRY(h, launch_rgb_beta_head(pl->ha, 0, pl->rg, h->head_taps, h->head_wgb, h->head_wbb, h->head_ntaps, xhat, pl->bsave, pl->n, st));
  return IAN_OK;
}

// IAN_simple's dec_out and tanh from the h3 planes
int run_dec_out(ian_handle* h, Plan* pl, float* xhat, cudaStream_t st) {
  ScopedTimer tm(h, T_DEC_OUT, st);
  if (h->path == IAN_PATH_TC) {
    float* one[1] = {xhat};
    LAUNCH_TRY(h, launch_dec_out_tc(pl->decout_maps, h->gather_dsts ? h->gather_dsts : one, h->gather_dsts ? h->gather_ndst : 1, pl->n, st));
  }
  else
    LAUNCH_TRY(h, launch_dec_out(pl->h3.p, pl->h3.plane, h->decout_wt, xhat, pl->n, st));
  return IAN_OK;
}

// zp must already hold the latent planes
int run_decode_from_planes(ian_handle* h, Plan* pl, float* xhat, cudaStream_t st) {
  int rc;
  for (int l : decoder_layers(h).fwd)
    if ((rc = run_gemm(h, pl, l, st)) != IAN_OK) return rc;
  return has_flow(h) ? run_head(h, pl, xhat, st) : run_dec_out(h, pl, xhat, st);
}

int run_decode(ian_handle* h, Plan* pl, const float* z, float* xhat, cudaStream_t st) {
  LAUNCH_TRY(h, launch_z_to_planes(z, pl->zp.p, pl->zp.plane, pl->n, st));
  return run_decode_from_planes(h, pl, xhat, st);
}

// decoder forward (from zp) + backward; leaves g (n,128 padded) in pl->gpad.  The loss seed is the box loss of
// boxes / target (brush gradients), or -- dxhat != NULL -- the caller's cotangent dL/dx_hat (n,3,64,64) over the whole
// frame (ian_decode_vjp_*); only the seed kernel differs between the two.
// param (IAN_simple, dxhat set): the parameter VJP's seed kernel, which also stores dec_out's seed image and dL/dh3.
int run_grad_core(ian_handle* h, Plan* pl, const int32_t* boxes, const float* target, int target_is_frame,
                  const float* dxhat, cudaStream_t st, bool param = false) {
  int rc;
  if ((rc = run_decode_from_planes(h, pl, pl->xhat, st)) != IAN_OK) return rc;
  if (has_flow(h)) {
    // the gradient is w.r.t. l_Z, the decoder's input (API.py:46: X_hat = get_output(l_out, {l_Z: Z})): no MADE/IAF backward
    {
      ScopedTimer tm(h, T_BRUSH_SEED, st);
      LAUNCH_TRY(h, launch_head_bwd_seed(pl->xhat, pl->rg, pl->bsave, boxes, target, target_is_frame, dxhat, pl->dpre, pl->n, st));
    }
    LAUNCH_TRY(h, launch_head_bwd(pl->rg, h->head_taps, h->head_wgb, h->head_wbb, h->head_ntaps, pl->dpre, pl->dha2.p,
                                  pl->dha2.plane, pl->n, st));
  } else {
    ScopedTimer tm(h, T_BRUSH_SEED, st);
    if (param)
      LAUNCH_TRY(h, launch_brush_param_seed_bwd(pl->xhat, dxhat, h->decout_wt, h->w[L_DEC_CONV3].scale, pl->h3.p, pl->d3.p,
                                                pl->d3.plane, pl->pseed, pl->dh3.p, pl->n, st));
    else
      LAUNCH_TRY(h, launch_brush_seed_bwd(pl->xhat, boxes, target, target_is_frame, dxhat, h->decout_wt, h->w[L_DEC_CONV3].scale,
                                          pl->h3.p, pl->d3.p, pl->d3.plane, pl->n, st));
  }
  for (int l : decoder_layers(h).bwd)
    if ((rc = run_gemm(h, pl, l, st)) != IAN_OK) return rc;
  return IAN_OK;
}

int check_ready(ian_handle* h, int n, const void* a, const void* b) {
  if (!h) return IAN_ERR_INVALID;
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "ian_finalize() has not been called");
  if (n <= 0) return fail(h, IAN_ERR_INVALID, "batch size must be positive (got %d)", n);
  if (!a || !b) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  return IAN_OK;
}

int validate_boxes(ian_handle* h, const int32_t* bx, int n) {
  for (int k = 0; k < n; ++k) {
    const int c1 = bx[4 * k], r1 = bx[4 * k + 1], c2 = bx[4 * k + 2], r2 = bx[4 * k + 3];
    if (c1 < 0 || r1 < 0 || c2 > 64 || r2 > 64 || c1 >= c2 || r1 >= r2)
      return fail(h, IAN_ERR_INVALID, "box %d = [c1=%d,r1=%d,c2=%d,r2=%d] is empty or outside the 64x64 frame", k, c1, r1, c2, r2);
  }
  return IAN_OK;
}

// ---- weight preparation --------------------------------------------------------------------------
const HostParam& P(ian_handle* h, const char* name) { return h->params[name]; }

// device buffer of `bytes`: allocated on first use (ian_finalize), overwritten in place afterwards (ian_update_param_host),
// so plans, tensor maps and captured graphs that hold the pointer stay valid
template <typename T>
int put_dev(ian_handle* h, T*& dst, const void* src, size_t bytes) {
  if (!dst) CUDA_TRY(h, cudaMalloc((void**)&dst, bytes));
  CUDA_TRY(h, cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
  return IAN_OK;
}

int upload_tiles(ian_handle* h, int l, const std::vector<float>& B, int ntiles, int Cout, int Cin) {
  DevWeights& w = h->w[l];
  const long long elems = (long long)ntiles * Cout * Cin;
  std::vector<uint16_t> planes((size_t)elems * 2);
  for (long long i = 0; i < elems; ++i) split_hi_lo(B[i], planes[i], planes[elems + i]);
  int rc = put_dev(h, w.b, planes.data(), planes.size() * 2);
  if (rc != IAN_OK) return rc;
  w.plane = elems; w.ntiles = ntiles; w.Cout = Cout; w.Cin = Cin;
  return IAN_OK;
}

int upload_gemm_weights(ian_handle* h, int l, const std::vector<float>& B, int ntiles, int Cout, int Cin,
                        const std::vector<float>& scale, const std::vector<float>& shift) {
  int rc = upload_tiles(h, l, B, ntiles, Cout, Cin);
  if (rc != IAN_OK) return rc;
  DevWeights& w = h->w[l];
  if ((rc = put_dev(h, w.scale, scale.data(), scale.size() * 4)) != IAN_OK) return rc;
  if (!shift.empty() && (rc = put_dev(h, w.shift, shift.data(), shift.size() * 4)) != IAN_OK) return rc;
  return IAN_OK;
}

// inference BatchNorm folded to y = x*scale + shift (lasagne batch_norm, IAN_simple.py:84-170)
void fold_bn(ian_handle* h, const std::string& name, int c, std::vector<float>& scale, std::vector<float>& shift) {
  const auto& be = P(h, (name + ".beta").c_str()).data;
  const auto& ga = P(h, (name + ".gamma").c_str()).data;
  const auto& me = P(h, (name + ".mean").c_str()).data;
  const auto& is = P(h, (name + ".inv_std").c_str()).data;
  scale.resize(c);
  shift.resize(c);
  for (int i = 0; i < c; ++i) {
    scale[i] = ga[i] * is[i];
    shift[i] = be[i] - me[i] * scale[i];
  }
}

int prepare_encoder(ian_handle* h) {
  int rc;
  std::vector<float> B, sc, sf;
  // enc_conv2..4: B[i*5+j][o][c] = W[o][c][i][j]
  struct CS { int l; const char* w; const char* bn; int Cout, Cin; } convs[] = {
      {L_ENC_CONV2, "enc_conv2.W", "bnorm2", 256, 128}, {L_ENC_CONV3, "enc_conv3.W", "bnorm3", 512, 256},
      {L_ENC_CONV4, "enc_conv4.W", "bnorm4", 1024, 512}};
  for (auto& c : convs) {
    const auto& W = P(h, c.w).data;
    B.assign((size_t)25 * c.Cout * c.Cin, 0.f);
    for (int o = 0; o < c.Cout; ++o)
      for (int ci = 0; ci < c.Cin; ++ci)
        for (int t = 0; t < 25; ++t) B[((size_t)t * c.Cout + o) * c.Cin + ci] = W[((size_t)o * c.Cin + ci) * 25 + t];
    fold_bn(h, c.bn, c.Cout, sc, sf);
    if ((rc = upload_gemm_weights(h, c.l, B, 25, c.Cout, c.Cin, sc, sf)) != IAN_OK) return rc;
  }
  {   // bnorm2..4's gamma | beta for the training-mode discriminator, which normalises with the batch's statistics
    std::vector<float> gb(2 * 1792);
    int off = 0;
    for (auto& c : convs) {
      const auto& ga = P(h, (std::string(c.bn) + ".gamma").c_str()).data;
      const auto& be = P(h, (std::string(c.bn) + ".beta").c_str()).data;
      std::copy(ga.begin(), ga.begin() + c.Cout, gb.begin() + off);
      std::copy(be.begin(), be.begin() + c.Cout, gb.begin() + 1792 + off);
      off += c.Cout;
    }
    if ((rc = put_dev(h, h->enc_bn_gb, gb.data(), gb.size() * sizeof(float))) != IAN_OK) return rc;
  }
  // enc_fc1: rows of W are flatten(NCHW) = c*16 + hw; our A is NHWC = hw*1024 + c.  Cout 1000 -> 1024.
  {
    const auto& W = P(h, "enc_fc1.W").data;
    B.assign((size_t)1024 * 16384, 0.f);
    for (int c = 0; c < 1024; ++c)
      for (int hw = 0; hw < 16; ++hw) {
        const float* src = &W[((size_t)c * 16 + hw) * 1000];
        for (int o = 0; o < 1000; ++o) B[(size_t)o * 16384 + hw * 1024 + c] = src[o];
      }
    fold_bn(h, "bnorm_enc_fc1", 1000, sc, sf);
    sc.resize(1024, 0.f);
    sf.resize(1024, 0.f);
    if ((rc = upload_gemm_weights(h, L_ENC_FC1, B, 1, 1024, 16384, sc, sf)) != IAN_OK) return rc;
  }
  // head: mu (cols 0..99) | logsigma (cols 100..199), Cout 200 -> 256, Cin 1000 -> 1024
  {
    const auto& Wm = P(h, "enc_mu.W").data;
    const auto& Wl = P(h, "enc_logsigma.W").data;
    B.assign((size_t)256 * 1024, 0.f);
    for (int k = 0; k < 1000; ++k)
      for (int o = 0; o < 100; ++o) {
        B[(size_t)o * 1024 + k] = Wm[(size_t)k * 100 + o];
        B[(size_t)(100 + o) * 1024 + k] = Wl[(size_t)k * 100 + o];
      }
    std::vector<float> s1, f1, s2, f2;
    fold_bn(h, "mu_bnorm", 100, s1, f1);
    fold_bn(h, "ls_bnorm", 100, s2, f2);
    sc.assign(256, 0.f);
    sf.assign(256, 0.f);
    for (int o = 0; o < 100; ++o) { sc[o] = s1[o]; sf[o] = f1[o]; sc[100 + o] = s2[o]; sf[100 + o] = f2[o]; }
    if ((rc = upload_gemm_weights(h, L_ENC_HEAD, B, 1, 256, 1024, sc, sf)) != IAN_OK) return rc;
  }
  // conv1: wt[(c*5+i)*5+j][o] = W[o][c][i][j]
  {
    const auto& W = P(h, "enc_conv1.W").data;
    std::vector<float> wt(75 * 128);
    for (int o = 0; o < 128; ++o)
      for (int k = 0; k < 75; ++k) wt[k * 128 + o] = W[o * 75 + k];
    CUDA_TRY(h, cudaMalloc((void**)&h->conv1_wt, wt.size() * 4));
    CUDA_TRY(h, cudaMemcpy(h->conv1_wt, wt.data(), wt.size() * 4, cudaMemcpyHostToDevice));
    const auto& b = P(h, "enc_conv1.b").data;
    CUDA_TRY(h, cudaMalloc((void**)&h->conv1_b, 128 * 4));
    CUDA_TRY(h, cudaMemcpy(h->conv1_b, b.data(), 128 * 4, cudaMemcpyHostToDevice));
    // tensor-core form: B[co][k] = W[co][c][i][j] (the reference layout flattened), K padded 75 -> 80, as three
    // [128 cout][64 k] blocks: hi of k < 64 | lo of k < 64 | tail (hi of k 64..79 at columns 0..15, lo at 16..31)
    std::vector<uint16_t> planes(3 * 128 * 64, 0);
    for (int o = 0; o < 128; ++o)
      for (int k = 0; k < 75; ++k) {
        if (k < 64)
          split_hi_lo(W[o * 75 + k], planes[o * 64 + k], planes[128 * 64 + o * 64 + k]);
        else
          split_hi_lo(W[o * 75 + k], planes[2 * 128 * 64 + o * 64 + (k - 64)], planes[2 * 128 * 64 + o * 64 + 16 + (k - 64)]);
      }
    CUDA_TRY(h, cudaMalloc((void**)&h->conv1_tc_wt, planes.size() * 2));
    CUDA_TRY(h, cudaMemcpy(h->conv1_tc_wt, planes.data(), planes.size() * 2, cudaMemcpyHostToDevice));
    char err[256] = {0};
    h->conv1_maps = conv1_build_maps(h->conv1_tc_wt, err, sizeof(err));
    if (!h->conv1_maps) return fail(h, IAN_ERR_CUDA, "enc_conv1: %s", err);
  }
  return IAN_OK;
}

// 5x5 stride-2 transposed conv weights W (Cin,Cout,5,5) -> forward tiles B[k][co][ci] = W[ci][co][k] (GEMM Cout padded to
// CoutPad with zero rows)
void deconv_fwd_tiles(const std::vector<float>& W, int Cin, int Cout, int CoutPad, std::vector<float>& B) {
  B.assign((size_t)25 * CoutPad * Cin, 0.f);
  for (int ci = 0; ci < Cin; ++ci)
    for (int co = 0; co < Cout; ++co)
      for (int t = 0; t < 25; ++t) B[((size_t)t * CoutPad + co) * Cin + ci] = W[((size_t)ci * Cout + co) * 25 + t];
}

// backward-data of the same layer: the gradient w.r.t. the deconv's INPUT is a stride-2 convolution of the output gradient
// with tiles B[k][ci][co] = W[ci][co][k] (GEMM Cout = the deconv's Cin, GEMM Cin = the deconv's Cout, padded to CoutPad)
void deconv_bwd_tiles(const std::vector<float>& W, int Cin, int Cout, int CoutPad, std::vector<float>& B) {
  B.assign((size_t)25 * Cin * CoutPad, 0.f);
  for (int ci = 0; ci < Cin; ++ci)
    for (int co = 0; co < Cout; ++co)
      for (int t = 0; t < 25; ++t) B[((size_t)t * Cin + ci) * CoutPad + co] = W[((size_t)ci * Cout + co) * 25 + t];
}
// transposed composite MDC tiles: comp [nt][F][C] -> [nt][C][F]
void transpose_tiles(const std::vector<float>& comp, int nt, int F, int C, std::vector<float>& out) {
  out.assign((size_t)nt * C * F, 0.f);
  for (int t = 0; t < nt; ++t)
    for (int f = 0; f < F; ++f)
      for (int c = 0; c < C; ++c) out[((size_t)t * C + c) * F + f] = comp[((size_t)t * F + f) * C + c];
}

// l_dec_fc2 (W (100, 16C)): the reference's column j = c*16 + hw is our NHWC column hw*C + c; K 100 -> 128.  Forward tiles
// B[col][k] (GEMM Cout 16C, Cin 128); backward (dz[k] = sum_col d[col] W[k][col]) tiles B[k][col] (GEMM Cout 128, Cin 16C).
void fc2_tiles(const std::vector<float>& W, int C, bool bwd, std::vector<float>& B) {
  const size_t cols = (size_t)16 * C;
  B.assign(cols * 128, 0.f);
  for (int c = 0; c < C; ++c)
    for (int hw = 0; hw < 16; ++hw) {
      const size_t j = (size_t)c * 16 + hw, col = hw * (size_t)C + c;
      for (int k = 0; k < 100; ++k) (bwd ? B[k * cols + col] : B[col * 128 + k]) = W[k * cols + j];
    }
}
// the reference's column of our column col (a per-feature vector of l_dec_fc2's output)
inline int fc2_ref_col(int col, int C) { return (col % C) * 16 + col / C; }

// ---- IAN_simple decoder: one derivation per parameter group, shared by ian_finalize and ian_update_param_host ----------
// Each writes every device buffer derived from its group: allocated by the first call, overwritten in place by later ones.
const char* kDecBn[4] = {"bnorm_dec_fc2", "bnorm_dc1", "bnorm_dc2", "bnorm_dc3"};
const int kDecBnC[4] = {16384, 512, 256, 128};
constexpr int kDecBnOff[4] = {0, 16384, 16896, 17152}, kDecBnTotal = 17280;   // the four BatchNorms' columns, concatenated
struct DecConv { int lf, lb; const char* w; int Cin, Cout; };
const DecConv kDecConv[3] = {{L_DEC_CONV1, L_BWD_CONV1, "dec_conv1.W", 1024, 512},
                             {L_DEC_CONV2, L_BWD_CONV2, "dec_conv2.W", 512, 256},
                             {L_DEC_CONV3, L_BWD_CONV3, "dec_conv3.W", 256, 128}};

// l_dec_fc2: forward and backward tiles (fc2_tiles), the backward with unit scale
int simple_fc2_weights(ian_handle* h, const std::vector<float>& W) {
  std::vector<float> B;
  fc2_tiles(W, 1024, false, B);
  int rc = upload_tiles(h, L_DEC_FC2, B, 1, 16384, 128);
  if (rc != IAN_OK) return rc;
  fc2_tiles(W, 1024, true, B);
  if ((rc = upload_tiles(h, L_BWD_FC2, B, 1, 128, 16384)) != IAN_OK) return rc;
  const std::vector<float> ones(128, 1.f);
  return put_dev(h, h->w[L_BWD_FC2].scale, ones.data(), ones.size() * 4);
}

// dec_conv k (W (Cin,Cout,5,5)): forward and backward-data tiles
int simple_conv_weights(ian_handle* h, int k, const std::vector<float>& W) {
  const DecConv& d = kDecConv[k];
  std::vector<float> B;
  deconv_fwd_tiles(W, d.Cin, d.Cout, d.Cout, B);
  int rc = upload_tiles(h, d.lf, B, 25, d.Cout, d.Cin);
  if (rc != IAN_OK) return rc;
  deconv_bwd_tiles(W, d.Cin, d.Cout, d.Cout, B);
  return upload_tiles(h, d.lb, B, 25, d.Cin, d.Cout);
}

// dec_out W (128,3,5,5): tensor-core form (decout_tc.cu, rows tap*3+co padded to 80, K-major over ci, bf16 hi|lo planes)
// and the FFMA form wt[tap][ci][co(4)] (SIMT forward, every seed kernel)
int simple_dec_out_weights(ian_handle* h, const std::vector<float>& W) {
  std::vector<uint16_t> planes(2 * 80 * 128, 0);
  std::vector<float> wt(25 * 128 * 4, 0.f);
  for (int ci = 0; ci < 128; ++ci)
    for (int co = 0; co < 3; ++co)
      for (int t = 0; t < 25; ++t) {
        const float w = W[(ci * 3 + co) * 25 + t];
        split_hi_lo(w, planes[(t * 3 + co) * 128 + ci], planes[80 * 128 + (t * 3 + co) * 128 + ci]);
        wt[(t * 128 + ci) * 4 + co] = w;
      }
  int rc = put_dev(h, h->decout_tc_wt, planes.data(), planes.size() * 2);
  if (rc != IAN_OK) return rc;
  return put_dev(h, h->decout_wt, wt.data(), wt.size() * 4);
}

// decoder BatchNorm k (0: bnorm_dec_fc2, 1..3: bnorm_dc1..3) from the host copy h->dec_bn[k]: the folded scale / shift of the
// layer's forward epilogue, the same scale in the backward-data epilogue of the layer above (bnorm_dc3's is read by the
// seed kernels from the forward buffer), and mean / inv_std on the device once the parameter VJP has used them
int simple_bn(ian_handle* h, int k) {
  const int C = kDecBnC[k];
  const auto& f = h->dec_bn[k];      // beta, gamma, mean, inv_std
  std::vector<float> sc(C), sf(C);
  for (int j = 0; j < C; ++j) {
    const int i = k == 0 ? fc2_ref_col(j, 1024) : j;
    sc[j] = f[1][i] * f[3][i];
    sf[j] = f[0][i] - f[2][i] * sc[j];
  }
  const int lf = k == 0 ? L_DEC_FC2 : kDecConv[k - 1].lf;
  int rc = put_dev(h, h->w[lf].scale, sc.data(), C * 4);
  if (rc != IAN_OK) return rc;
  if ((rc = put_dev(h, h->w[lf].shift, sf.data(), C * 4)) != IAN_OK) return rc;
  if (k < 3 && (rc = put_dev(h, h->w[kDecConv[k].lb].scale, sc.data(), C * 4)) != IAN_OK) return rc;
  {   // gamma | beta in the library's column order for the training-mode decoder, which normalises with the batch's statistics
    if (!h->dec_bn_gb) CUDA_TRY(h, cudaMalloc((void**)&h->dec_bn_gb, 2 * kDecBnTotal * sizeof(float)));
    for (int j = 0; j < C; ++j) {
      const int i = k == 0 ? fc2_ref_col(j, 1024) : j;
      sc[j] = f[1][i];
      sf[j] = f[0][i];
    }
    CUDA_TRY(h, cudaMemcpy(h->dec_bn_gb + kDecBnOff[k], sc.data(), C * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->dec_bn_gb + kDecBnTotal + kDecBnOff[k], sf.data(), C * 4, cudaMemcpyHostToDevice));
  }
  if (h->dec_bn_stats[k][0]) {
    if ((rc = put_dev(h, h->dec_bn_stats[k][0], f[2].data(), C * 4)) != IAN_OK) return rc;
    if ((rc = put_dev(h, h->dec_bn_stats[k][1], f[3].data(), C * 4)) != IAN_OK) return rc;
  }
  return IAN_OK;
}

int prepare_simple_decoder(ian_handle* h) {
  for (int k = 0; k < 4; ++k)
    for (int f = 0; f < 4; ++f) h->dec_bn[k][f] = P(h, (std::string(kDecBn[k]) + "." + kBnFields[f]).c_str()).data;
  int rc = simple_fc2_weights(h, P(h, "l_dec_fc2.W").data);
  for (int k = 0; k < 3 && rc == IAN_OK; ++k) rc = simple_conv_weights(h, k, P(h, kDecConv[k].w).data);
  for (int k = 0; k < 4 && rc == IAN_OK; ++k) rc = simple_bn(h, k);
  if (rc == IAN_OK) rc = simple_dec_out_weights(h, P(h, "dec_out.W").data);
  return rc;
}

// composite MDC weights (reference layers.py:207-258): per distinct offset one [F][C] matrix
//   base 3x3: W[f,c,i,j]*coeff_base[f] at (i-1, j-1);  scale 0: mean_ij(W)*coeff_1x1[f] at (0,0);
//   scale s: W[f,c,i,j]*coeff_s[f] at ((i-1)s, (j-1)s)
void mdc_composite(ian_handle* h, const std::string& name, int F, int C, const std::vector<int>& scales,
                   std::vector<float>& comp /*[ntaps][F][C]*/) {
  const auto off = mdc_offsets(scales);
  const auto& W = P(h, (name + "W").c_str()).data;
  comp.assign(off.size() * (size_t)F * C, 0.f);
  auto tile_of = [&](int dy, int dx) { for (size_t t = 0; t < off.size(); ++t) if (off[t].first == dy && off[t].second == dx) return (int)t; return -1; };
  auto put = [&](int s, const std::vector<float>& coeff) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const int t = tile_of((i - 1) * s, (j - 1) * s);
        for (int f = 0; f < F; ++f)
          for (int c = 0; c < C; ++c) comp[((size_t)t * F + f) * C + c] += W[(((size_t)f * C + c) * 3 + i) * 3 + j] * coeff[f];
      }
  };
  put(1, P(h, (name + "_coeff_base").c_str()).data);
  for (int s : scales) {
    if (s == 0) {
      const auto& coeff = P(h, (name + "_coeff_1x1").c_str()).data;
      const int t = tile_of(0, 0);
      for (int f = 0; f < F; ++f)
        for (int c = 0; c < C; ++c) {
          float m = 0.f;
          for (int k = 0; k < 9; ++k) m += W[((size_t)f * C + c) * 9 + k];
          comp[((size_t)t * F + f) * C + c] += (m / 9.f) * coeff[f];
        }
    } else {
      put(s, P(h, (name + "_coeff_" + std::to_string(s)).c_str()).data);
    }
  }
}

// MADE connectivity (reference mask_generator.py:29-38,93-94 as API.IAN leaves it after reset("Once")): with ordering o,
// layer connectivities are input = o + 1, hidden = 1, output = o and a weight (i -> j) survives iff
// conn_in[i] <= conn_out[j].  which: 0 = `_input` (input -> hidden), 1 = `_output_W` (hidden -> output),
// 2 = `_output_D` (input -> output, direct).  Integer comparisons only: W * M is bit-exact.
inline bool made_keep(const int32_t* o, int which, int i, int j) {
  return which == 0 ? (o[i] + 1 <= 1) : which == 1 ? (1 <= o[j]) : (o[i] + 1 <= o[j]);
}

int prepare_made(ian_handle* h) {
  // ---- MADE (layers.py:653-853): masks from the ordering (mask_generator.py:93-94; SURVEY Appendix D), integer
  // comparisons, multiplied into the float32 weights here on the host (bit-exact W*M)
  {
    if (h->made_ordering.size() != 100) return fail(h, IAN_ERR_STATE, "ian_set_made_ordering() must precede ian_finalize() for the full IAN");
    const auto& o = h->made_ordering;
    std::vector<float> mw(2 * 3 * 10000), mb(2 * 3 * 100);
    const char* nets[2] = {"l_IAF_mu", "l_IAF_ls"};
    const char* subs[3] = {"_input", "_output_W", "_output_D"};
    for (int net = 0; net < 2; ++net)
      for (int m = 0; m < 3; ++m) {
        const auto& W = P(h, (std::string(nets[net]) + subs[m] + ".W").c_str()).data;
        const auto& b = P(h, (std::string(nets[net]) + subs[m] + ".b").c_str()).data;
        for (int i = 0; i < 100; ++i)
          for (int j = 0; j < 100; ++j) {
            const bool keep = made_keep(o.data(), m, i, j);
            mw[((net * 3 + m) * 100 + i) * 100 + j] = keep ? W[i * 100 + j] : 0.f;
          }
        for (int j = 0; j < 100; ++j) mb[(net * 3 + m) * 100 + j] = b[j];
      }
    CUDA_TRY(h, cudaMalloc((void**)&h->made_w, mw.size() * 4));
    CUDA_TRY(h, cudaMemcpy(h->made_w, mw.data(), mw.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMalloc((void**)&h->made_b, mb.size() * 4));
    CUDA_TRY(h, cudaMemcpy(h->made_b, mb.data(), mb.size() * 4, cudaMemcpyHostToDevice));
  }
  return IAN_OK;
}

// RGB-Beta head weights for a feature map with C real channels (128 for IAN.py, 64 for IANv1.py) stored 128 wide
int prepare_head(ian_handle* h, int C, const std::vector<float>& scale_below /*BN scale of the feature map (128 wide)*/) {
  int rc;
  std::vector<float> B, sc, comp;
  // ---- RGB-Beta head (IAN.py:183-207): the three 128->2 MDC convs as one 16-row tile [R | G_a | B_a | 0...]
  {
    const std::vector<int> hs = {2, 3, 4};
    const auto off = mdc_offsets(hs);
    const int nt = (int)off.size();
    if (nt * 6 != 198) return fail(h, IAN_ERR_STATE, "unexpected head tap count %d", nt);
    // one weight tile [256 rows][128]: row t*6 + (2k+f) = composite tap t of filter f of conv k in {R, G_a, B_a}
    B.assign((size_t)256 * 128, 0.f);
    const char* names[3] = {"R", "G_a", "B_a"};
    for (int k = 0; k < 3; ++k) {
      mdc_composite(h, names[k], 2, C, hs, comp);
      for (int t = 0; t < nt; ++t)
        for (int f = 0; f < 2; ++f)
          for (int c = 0; c < C; ++c) B[((size_t)(t * 6 + 2 * k + f)) * 128 + c] = comp[((size_t)t * 2 + f) * C + c];
    }
    sc.assign(256, 1.f);
    if ((rc = upload_gemm_weights(h, F_HEAD, B, 1, 256, 128, sc, {})) != IAN_OK) return rc;
    // backward: dh[c] = sum_k A2[k] * B[k][c], k = t*6 + (2 conv + filter): the transposed tile, GEMM Cout = 128, Cin = 256
    std::vector<float> Bt((size_t)128 * 256, 0.f);
    for (int k = 0; k < 256; ++k)
      for (int c = 0; c < 128; ++c) Bt[(size_t)c * 256 + k] = B[(size_t)k * 128 + c];
    if ((rc = upload_gemm_weights(h, F_BWD_HEAD, Bt, 1, 128, 256, scale_below, {})) != IAN_OK) return rc;
    std::vector<int> taps(nt * 2);
    for (int t = 0; t < nt; ++t) { taps[2 * t] = off[t].first; taps[2 * t + 1] = off[t].second; }
    CUDA_TRY(h, cudaMalloc((void**)&h->head_taps, taps.size() * 4));
    CUDA_TRY(h, cudaMemcpy(h->head_taps, taps.data(), taps.size() * 4, cudaMemcpyHostToDevice));
    h->head_ntaps = nt;
    // fused head (head_tc.cu): taps sorted by row offset (stable), per conv k one 80-row tile: row = sorted tap * 2 + filter
    {
      std::vector<int> order;
      int pos = 0;
      for (int dy = -4; dy <= 4; ++dy) {
        h->head_dy_start[dy + 4] = pos;
        for (int t = 0; t < nt; ++t)
          if (off[t].first == dy) { order.push_back(t); h->head_dx[pos++] = off[t].second; }
      }
      h->head_dy_start[9] = pos;
      if (pos != 33) return fail(h, IAN_ERR_STATE, "head taps do not fit the [-4,4] row-offset window");
      // head_tc.cu's gather uses the analytic form of this table: dy != 0 -> dx in {-|dy|, 0, |dy|}; dy = 0 -> the nine offsets
      // in the order base 3x3, then dilations 2, 3, 4 (mdc_offsets' insertion order).  Refuse anything else.
      const int dx0[9] = {-1, 0, 1, -2, 2, -3, 3, -4, 4};
      for (int dy = -4; dy <= 4; ++dy) {
        const int j0 = h->head_dy_start[dy + 4], cnt = h->head_dy_start[dy + 5] - j0;
        bool ok = cnt == (dy == 0 ? 9 : 3) && j0 == (dy < 0 ? 3 * (dy + 4) : dy == 0 ? 12 : 21 + 3 * (dy - 1));
        for (int e = 0; ok && e < cnt; ++e) {
          const int a = dy < 0 ? -dy : dy;
          ok = h->head_dx[j0 + e] == (dy == 0 ? dx0[e] : (e - 1) * a);
        }
        if (!ok) return fail(h, IAN_ERR_STATE, "RGB-head tap set differs from the scales-[2,3,4] MDC layout head_tc.cu assumes");
      }
      std::vector<uint16_t> planes((size_t)2 * 3 * 80 * 128, 0);
      const size_t plane = (size_t)3 * 80 * 128;
      for (int k = 0; k < 3; ++k)
        for (int j = 0; j < 33; ++j)
          for (int f = 0; f < 2; ++f)
            for (int c = 0; c < 128; ++c) {
              const size_t row = (size_t)k * 80 + j * 2 + f;
              split_hi_lo(B[((size_t)(order[j] * 6 + 2 * k + f)) * 128 + c], planes[row * 128 + c], planes[plane + row * 128 + c]);
            }
      CUDA_TRY(h, cudaMalloc((void**)&h->head_tc_wt, planes.size() * 2));
      CUDA_TRY(h, cudaMemcpy(h->head_tc_wt, planes.data(), planes.size() * 2, cudaMemcpyHostToDevice));
    }
    mdc_composite(h, "G_b", 2, 2, hs, comp);             // [nt][2 out][2 in]
    CUDA_TRY(h, cudaMalloc((void**)&h->head_wgb, comp.size() * 4));
    CUDA_TRY(h, cudaMemcpy(h->head_wgb, comp.data(), comp.size() * 4, cudaMemcpyHostToDevice));
    mdc_composite(h, "B_b", 2, 4, hs, comp);             // [nt][2 out][4 in]
    CUDA_TRY(h, cudaMalloc((void**)&h->head_wbb, comp.size() * 4));
    CUDA_TRY(h, cudaMemcpy(h->head_wbb, comp.data(), comp.size() * 4, cudaMemcpyHostToDevice));
  }
  return IAN_OK;
}

// IANv1 decoder weights (IANv1.py:125-175)
int prepare_v1_decoder(ian_handle* h) {
  int rc;
  std::vector<float> B, sc, sf;
  if ((rc = prepare_made(h)) != IAN_OK) return rc;
  {   // l_dec_fc2: dense 100 -> 16384 + bias, NO nonlinearity
    const auto& b = P(h, "l_dec_fc2.b").data;
    fc2_tiles(P(h, "l_dec_fc2.W").data, 1024, false, B);
    sc.assign(16384, 1.f);
    sf.resize(16384);
    for (int col = 0; col < 16384; ++col) sf[col] = b[fc2_ref_col(col, 1024)];
    if ((rc = upload_gemm_weights(h, L_DEC_FC2, B, 1, 16384, 128, sc, sf)) != IAN_OK) return rc;
  }
  struct St { int l; const char* w; const char* bn; int Cin, Cout; } sts[3] = {
      {L_DEC_CONV1, "dec_conv1.W", "bnorm_dc1", 1024, 512}, {L_DEC_CONV2, "dec_conv2.W", "bnorm_dc2", 512, 256},
      {L_DEC_CONV3, "dec_conv3.W", "bnorm_dc3", 256, 128}};
  for (const St& s : sts) {
    deconv_fwd_tiles(P(h, s.w).data, s.Cin, s.Cout, s.Cout, B);
    fold_bn(h, s.bn, s.Cout, sc, sf);
    if ((rc = upload_gemm_weights(h, s.l, B, 25, s.Cout, s.Cin, sc, sf)) != IAN_OK) return rc;
  }
  {   // dec_conv4: 128 -> 64 channels, stored 128 wide: channels 64..127 have zero weights, scale and shift (relu(0) = 0)
    deconv_fwd_tiles(P(h, "dec_conv4.W").data, 128, 64, 128, B);
    fold_bn(h, "bnorm_dc4", 64, sc, sf);
    sc.resize(128, 0.f);
    sf.resize(128, 0.f);
    if ((rc = upload_gemm_weights(h, F_DEC_CONV4, B, 25, 128, 128, sc, sf)) != IAN_OK) return rc;
  }
  // ---- brush backward: each backward GEMM's epilogue applies the BN scale (and the ReLU mask) of the layer BELOW it
  std::vector<float> s4 = sc, s3, s2, s1, f_;              // s4: bnorm_dc4 scale (64 real channels, padded with zeros)
  fold_bn(h, "bnorm_dc3", 128, s3, f_); fold_bn(h, "bnorm_dc2", 256, s2, f_); fold_bn(h, "bnorm_dc1", 512, s1, f_);
  deconv_bwd_tiles(P(h, "dec_conv4.W").data, 128, 64, 128, B);
  if ((rc = upload_gemm_weights(h, F_BWD_CONV4, B, 25, 128, 128, s3, {})) != IAN_OK) return rc;
  deconv_bwd_tiles(P(h, "dec_conv3.W").data, 256, 128, 128, B);
  if ((rc = upload_gemm_weights(h, L_BWD_CONV3, B, 25, 256, 128, s2, {})) != IAN_OK) return rc;
  deconv_bwd_tiles(P(h, "dec_conv2.W").data, 512, 256, 256, B);
  if ((rc = upload_gemm_weights(h, L_BWD_CONV2, B, 25, 512, 256, s1, {})) != IAN_OK) return rc;
  deconv_bwd_tiles(P(h, "dec_conv1.W").data, 1024, 512, 512, B);
  if ((rc = upload_gemm_weights(h, L_BWD_CONV1, B, 25, 1024, 512, std::vector<float>(1024, 1.f), {})) != IAN_OK) return rc;
  fc2_tiles(P(h, "l_dec_fc2.W").data, 1024, true, B);
  if ((rc = upload_gemm_weights(h, L_BWD_FC2, B, 1, 128, 16384, std::vector<float>(128, 1.f), {})) != IAN_OK) return rc;
  return prepare_head(h, 64, s4);
}

int prepare_full_decoder(ian_handle* h) {
  int rc;
  std::vector<float> B, sc, sf, comp;
  if ((rc = prepare_made(h)) != IAN_OK) return rc;
  // ---- l_dec_fc2: dense 100 -> 8192 + bias, lrelu (IAN.py:129-134)
  {
    const auto& b = P(h, "l_dec_fc2.b").data;
    fc2_tiles(P(h, "l_dec_fc2.W").data, 512, false, B);
    sc.assign(8192, 1.f);
    sf.resize(8192);
    for (int col = 0; col < 8192; ++col) sf[col] = b[fc2_ref_col(col, 512)];
    if ((rc = upload_gemm_weights(h, F_DEC_FC2, B, 1, 8192, 128, sc, sf)) != IAN_OK) return rc;
  }
  // ---- deconvs + MDBLOCKs (IAN.py:139-171)
  struct St { int dconv, mda, mdb; const char* w; const char* blk; int Cin, Cout; std::vector<int> scales; };
  const St sts[3] = {{F_DEC_CONV1, F_MD1A, F_MD1B, "dec_conv1.W", "dec_conv2a", 512, 512, {0, 2}},
                     {F_DEC_CONV2, F_MD2A, F_MD2B, "dec_conv2.W", "dec_conv3a", 512, 256, {0, 2, 3}},
                     {F_DEC_CONV3, F_MD3A, F_MD3B, "dec_conv3.W", "dec_conv4a", 256, 128, {0, 2, 3}}};
  for (const St& s : sts) {
    deconv_fwd_tiles(P(h, s.w).data, s.Cin, s.Cout, s.Cout, B);
    fold_bn(h, std::string(s.blk) + "bnorm0", s.Cout, sc, sf);
    if ((rc = upload_gemm_weights(h, s.dconv, B, 25, s.Cout, s.Cin, sc, sf)) != IAN_OK) return rc;
    const int nt = (int)mdc_offsets(s.scales).size();
    mdc_composite(h, s.blk, s.Cout, s.Cout, s.scales, comp);
    fold_bn(h, std::string(s.blk) + "bnorm1", s.Cout, sc, sf);
    if ((rc = upload_gemm_weights(h, s.mda, comp, nt, s.Cout, s.Cout, sc, sf)) != IAN_OK) return rc;
    mdc_composite(h, std::string(s.blk) + "2", s.Cout, s.Cout, s.scales, comp);
    fold_bn(h, std::string(s.blk) + "bnorm2", s.Cout, sc, sf);
    if ((rc = upload_gemm_weights(h, s.mdb, comp, nt, s.Cout, s.Cout, sc, sf)) != IAN_OK) return rc;
  }
  deconv_fwd_tiles(P(h, "dec_conv4.W").data, 128, 128, 128, B);
  fold_bn(h, "bnorm_dc4", 128, sc, sf);
  if ((rc = upload_gemm_weights(h, F_DEC_CONV4, B, 25, 128, 128, sc, sf)) != IAN_OK) return rc;
  if ((rc = prepare_head(h, 128, sc)) != IAN_OK) return rc;
  // ---- brush backward (see wire_decoder_full): every backward GEMM's epilogue applies the BN scale of the activation it lands on
  struct Bk { int dconv, mdb, mda; const char* w_above; int Cin_above, Cout_above; const char* blk; int C; std::vector<int> scales; };
  // dconv = backward-data of the deconv ABOVE block `blk` (w_above: (Cin_above = this block's C, Cout_above))
  const Bk bks[3] = {{F_BWD_CONV4, F_BWD_MD3B, F_BWD_MD3A, "dec_conv4.W", 128, 128, "dec_conv4a", 128, {0, 2, 3}},
                     {F_BWD_CONV3, F_BWD_MD2B, F_BWD_MD2A, "dec_conv3.W", 256, 128, "dec_conv3a", 256, {0, 2, 3}},
                     {F_BWD_CONV2, F_BWD_MD1B, F_BWD_MD1A, "dec_conv2.W", 512, 256, "dec_conv2a", 512, {0, 2}}};
  std::vector<float> s0, s1, s2, f_, Bt;
  for (const Bk& b : bks) {
    fold_bn(h, std::string(b.blk) + "bnorm0", b.C, s0, f_);
    fold_bn(h, std::string(b.blk) + "bnorm1", b.C, s1, f_);
    fold_bn(h, std::string(b.blk) + "bnorm2", b.C, s2, f_);
    deconv_bwd_tiles(P(h, b.w_above).data, b.Cin_above, b.Cout_above, b.Cout_above, B);
    if ((rc = upload_gemm_weights(h, b.dconv, B, 25, b.Cin_above, b.Cout_above, s2, {})) != IAN_OK) return rc;
    const int nt = (int)mdc_offsets(b.scales).size();
    mdc_composite(h, std::string(b.blk) + "2", b.C, b.C, b.scales, comp);
    transpose_tiles(comp, nt, b.C, b.C, Bt);
    if ((rc = upload_gemm_weights(h, b.mdb, Bt, nt, b.C, b.C, s1, {})) != IAN_OK) return rc;
    mdc_composite(h, b.blk, b.C, b.C, b.scales, comp);
    transpose_tiles(comp, nt, b.C, b.C, Bt);
    if ((rc = upload_gemm_weights(h, b.mda, Bt, nt, b.C, b.C, s0, {})) != IAN_OK) return rc;
  }
  deconv_bwd_tiles(P(h, "dec_conv1.W").data, 512, 512, 512, B);
  if ((rc = upload_gemm_weights(h, F_BWD_CONV1, B, 25, 512, 512, std::vector<float>(512, 1.f), {})) != IAN_OK) return rc;
  fc2_tiles(P(h, "l_dec_fc2.W").data, 512, true, B);
  return upload_gemm_weights(h, F_BWD_FC2, B, 1, 128, 8192, std::vector<float>(128, 1.f), {});
}

// stream memory operations (driver API, fetched through the runtime): the free / pushed flag handshake of the pipelined
// all-gather runs as cuStreamWriteValue32 / cuStreamWaitValue32 on peer-mapped memory -- no kernel, hence no SM slot
typedef CUresult (*StreamWrite32Fn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
typedef CUresult (*StreamWait32Fn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
struct MemOps { StreamWrite32Fn write = nullptr; StreamWait32Fn wait = nullptr; };
inline const MemOps& memops() {
  static MemOps m;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void *pw = nullptr, *pq = nullptr;
    cudaDriverEntryPointQueryResult q1, q2;
    if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &pw, cudaEnableDefault, &q1) == cudaSuccess && q1 == cudaDriverEntryPointSuccess &&
        cudaGetDriverEntryPoint("cuStreamWaitValue32", &pq, cudaEnableDefault, &q2) == cudaSuccess && q2 == cudaDriverEntryPointSuccess) {
      m.write = reinterpret_cast<StreamWrite32Fn>(pw);
      m.wait = reinterpret_cast<StreamWait32Fn>(pq);
    }
  }
  return m;
}

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

template <typename F>
int for_chunks(ian_handle* h, int n, F&& f) {
  for (int off = 0; off < n; off += h->max_chunk) {
    const int cn = (n - off < h->max_chunk) ? n - off : h->max_chunk;
    Plan* pl = nullptr;
    int rc = get_plan(h, cn, &pl);
    if (rc != IAN_OK) return rc;
    if ((rc = f(pl, off, cn)) != IAN_OK) return rc;
  }
  return IAN_OK;
}

// The interactive calls (NPE: batch 1) are launch-bound: ~20-40 kernels of a few microseconds each.  The kernel
// sequence of a host entry point depends only on the plan (fixed buffers, fixed tensor maps) and a few scalars, so it is
// captured once per (plan, entry point, key) and replayed with one cudaGraphLaunch; the H2D/D2H copies of the
// caller's buffers stay outside the graph.  Large batches are not launch-bound (and may schedule stream-K, whose
// epoch is a kernel argument): they keep plain launches.  kGraphMaxBatch is defined above run_gemm, which also reads it.

template <typename F>
int run_graphed(ian_handle* h, Plan* pl, int slot, uint64_t key, cudaStream_t st, F&& body) {
  if (!h->graphs || h->timing || h->path != IAN_PATH_TC || pl->n > kGraphMaxBatch || st != h->stream || h->gather_dsts)
    return body();
  Plan::GraphSlot& gs = pl->graph[slot];
  key = key * 4 + (uint64_t)(h->passes == 1 ? 1 : 0) + 2;      // +2: a valid key is never 0
  if (gs.exec && gs.key != key) {
    cudaGraphExecDestroy(gs.exec);
    gs.exec = nullptr;
  }
  if (!gs.exec) {
    const int64_t l0 = h->launches;
    CUDA_TRY(h, cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed));
    h->capturing = true;
    const int r = body();
    h->capturing = false;
    cudaGraph_t graph = nullptr;
    const cudaError_t e = cudaStreamEndCapture(st, &graph);
    gs.launches = h->launches - l0;
    h->launches = l0;
    if (r != IAN_OK) { if (graph) cudaGraphDestroy(graph); return r; }
    if (e != cudaSuccess) return fail(h, IAN_ERR_CUDA, "cudaStreamEndCapture failed: %s", cudaGetErrorString(e));
    const cudaError_t ei = cudaGraphInstantiate(&gs.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ei != cudaSuccess) { gs.exec = nullptr; return fail(h, IAN_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ei)); }
    gs.key = key;
  }
  CUDA_TRY(h, cudaGraphLaunch(gs.exec, st));
  h->launches += gs.launches;
  return IAN_OK;
}

inline uint64_t float_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

// ---- encoder vector-Jacobian product -------------------------------------------------------------
// dx = (dz/dx)^T dz through the encoder (and, on IAN.py / IANv1.py, the MADE/IAF flow).  The adjoint of a layer whose
// forward tile is B[t][co][ci] is the tap-GEMM with tiles B'[t'][ci][co]: for the dense layers t' = t; for the 5x5
// stride-2 convolutions y[p] = sum_i x[2p+i-2] W[i], the adjoint dx[2q+r] = sum_d dy[q+d] W[2+r-2d] is the decoder's
// transposed convolution (taps_deconv_s2, tile 2+2d-r) on the flipped tile t' = 24 - t.  ian_finalize has dropped the
// host parameters by now, so the tiles are permuted on the device from the forward ones: a hi|lo split is per element,
// so a permuted pair of planes is bit for bit what splitting the re-laid float32 weights would give.
// Each backward GEMM's epilogue applies the derivative of the activation it lands on (LeakyRectify(0.2) as the mask
// slope on the stored forward activation) times that layer's BatchNorm scale.
int ensure_enc_vjp_weights(ian_handle* h) {
  if (h->conv1_bwd_wt && h->conv1_bwd_tc_wt) return IAN_OK;
  cudaStream_t st = h->stream;
  struct Perm { int lb, lf, flip; const float* scale_src; int scale_len, repeat; } perms[] = {
      {E_BWD_HEAD, L_ENC_HEAD, 0, nullptr, 1024, 1},                   // 256 -> 1024; enc_fc1's derivative: enc_fc1_bwd_kernel
      {E_BWD_FC1, L_ENC_FC1, 0, h->w[L_ENC_CONV4].scale, 1024, 16},   // 1024 -> 16384 = (4,4,1024) NHWC: bnorm4 scale, per column
      {E_BWD_CONV4, L_ENC_CONV4, 1, h->w[L_ENC_CONV3].scale, 512, 1},  // -> a3: bnorm3
      {E_BWD_CONV3, L_ENC_CONV3, 1, h->w[L_ENC_CONV2].scale, 256, 1},  // -> a2: bnorm2
      {E_BWD_CONV2, L_ENC_CONV2, 1, nullptr, 128, 1}};                 // -> a1: conv1 has a bias and no BatchNorm
  for (const Perm& p : perms) {
    const DevWeights& f = h->w[p.lf];
    DevWeights& b = h->w[p.lb];
    if (!b.b) {
      CUDA_TRY(h, cudaMalloc((void**)&b.b, (size_t)f.plane * 2 * sizeof(__nv_bfloat16)));
      LAUNCH_TRY(h, launch_permute_tiles(f.b, f.plane, b.b, f.ntiles, f.Cout, f.Cin, p.flip, st));
      b.plane = f.plane; b.ntiles = f.ntiles; b.Cout = f.Cin; b.Cin = f.Cout;
    }
    if (!b.scale) {
      CUDA_TRY(h, cudaMalloc((void**)&b.scale, (size_t)p.scale_len * p.repeat * sizeof(float)));
      if (p.scale_src) {
        for (int r = 0; r < p.repeat; ++r)
          CUDA_TRY(h, cudaMemcpyAsync(b.scale + (size_t)r * p.scale_len, p.scale_src, (size_t)p.scale_len * sizeof(float),
                                      cudaMemcpyDeviceToDevice, st));
      } else {
        const std::vector<float> ones((size_t)p.scale_len, 1.f);
        CUDA_TRY(h, cudaMemcpyAsync(b.scale, ones.data(), ones.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        CUDA_TRY(h, cudaStreamSynchronize(st));
      }
    }
  }
  // enc_conv1's adjoint in dec_out's layout: wt[t][o][c] = W1[o][c][24 - t], from conv1_wt[(c*25 + t)*128 + o]
  std::vector<float> w1(75 * 128), wt(25 * 128 * 4, 0.f);
  CUDA_TRY(h, cudaMemcpyAsync(w1.data(), h->conv1_wt, w1.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaStreamSynchronize(st));
  for (int t = 0; t < 25; ++t)
    for (int o = 0; o < 128; ++o)
      for (int c = 0; c < 3; ++c) wt[((size_t)t * 128 + o) * 4 + c] = w1[((size_t)c * 25 + 24 - t) * 128 + o];
  // tensor-core form (decout_tc.cu's layout): rows tap*3 + c (75, padded to 80), K-major over o; bf16 hi|lo planes
  std::vector<uint16_t> planes(2 * 80 * 128, 0);
  for (int t = 0; t < 25; ++t)
    for (int c = 0; c < 3; ++c)
      for (int o = 0; o < 128; ++o)
        split_hi_lo(wt[((size_t)t * 128 + o) * 4 + c], planes[(t * 3 + c) * 128 + o], planes[80 * 128 + (t * 3 + c) * 128 + o]);
  if (!h->conv1_bwd_tc_wt) {
    CUDA_TRY(h, cudaMalloc((void**)&h->conv1_bwd_tc_wt, planes.size() * 2));
    CUDA_TRY(h, cudaMemcpyAsync(h->conv1_bwd_tc_wt, planes.data(), planes.size() * 2, cudaMemcpyHostToDevice, st));
  }
  if (!h->conv1_bwd_wt) {
    CUDA_TRY(h, cudaMalloc((void**)&h->conv1_bwd_wt, wt.size() * sizeof(float)));
    CUDA_TRY(h, cudaMemcpyAsync(h->conv1_bwd_wt, wt.data(), wt.size() * sizeof(float), cudaMemcpyHostToDevice, st));
  }
  CUDA_TRY(h, cudaStreamSynchronize(st));
  return IAN_OK;
}

int ensure_enc_vjp_plan(ian_handle* h, Plan* pl) {
  if (pl->evjp) return IAN_OK;
  int rc;
  if ((rc = ensure_enc_vjp_weights(h)) != IAN_OK) return rc;
  const int n = pl->n;
  const long long N = n;
  if ((rc = alloc_planes(h, pl, pl->eh, N * 256)) != IAN_OK) return rc;
  if ((rc = alloc_planes(h, pl, pl->ef1, N * 1024)) != IAN_OK) return rc;
  if ((rc = alloc_planes(h, pl, pl->e4, N * 16384)) != IAN_OK) return rc;
  if ((rc = alloc_planes(h, pl, pl->e3, N * 8 * 8 * 512)) != IAN_OK) return rc;
  if ((rc = alloc_planes(h, pl, pl->e2, N * 16 * 16 * 256)) != IAN_OK) return rc;
  if ((rc = alloc_planes(h, pl, pl->e1, N * 32 * 32 * 128)) != IAN_OK) return rc;
  if ((rc = alloc_buf(h, pl, pl->edz, N * 100)) != IAN_OK) return rc;
  if ((rc = alloc_buf(h, pl, pl->edzi, N * 100)) != IAN_OK) return rc;
  if ((rc = alloc_buf(h, pl, pl->eg, N * 1024)) != IAN_OK) return rc;
  TapGemm* g = pl->g;
  auto mask = [&](int l, const Planes& m, const Planes& out) {
    g[l].act = ACT_MASK; g[l].mask = m.p; g[l].mask_slope = 0.2f; g[l].out = out.p; g[l].out_plane = out.plane;
  };
  set_io(g[E_BWD_HEAD], pl->eh, n, 1, 1, 256, 1, 1, h->w[E_BWD_HEAD], 1, 1); taps_dense(g[E_BWD_HEAD]);
  g[E_BWD_HEAD].act = ACT_NONE; g[E_BWD_HEAD].out_f32 = pl->eg;
  set_io(g[E_BWD_FC1], pl->ef1, n, 1, 1, 1024, 1, 1, h->w[E_BWD_FC1], 1, 1); taps_dense(g[E_BWD_FC1]);
  mask(E_BWD_FC1, pl->a4, pl->e4);                      // a4 (n,4,4,1024) NHWC is the (n,16384) output's geometry
  set_io(g[E_BWD_CONV4], pl->e4, n, 4, 4, 1024, 4, 4, h->w[E_BWD_CONV4], 8, 8); taps_deconv_s2(g[E_BWD_CONV4]);
  mask(E_BWD_CONV4, pl->a3, pl->e3);
  set_io(g[E_BWD_CONV3], pl->e3, n, 8, 8, 512, 8, 8, h->w[E_BWD_CONV3], 16, 16); taps_deconv_s2(g[E_BWD_CONV3]);
  mask(E_BWD_CONV3, pl->a2, pl->e2);
  set_io(g[E_BWD_CONV2], pl->e2, n, 16, 16, 256, 16, 16, h->w[E_BWD_CONV2], 32, 32); taps_deconv_s2(g[E_BWD_CONV2]);
  mask(E_BWD_CONV2, pl->a1, pl->e1);
  // the chain's own split-K slabs: the plan's other layers keep theirs
  if ((rc = finish_maps(h, pl, kEncoderBwd)) != IAN_OK) return rc;
  {   // both paths: ian_set_path may switch a live handle
    char err[256] = {0};
    pl->conv1_bwd_maps = decout_build_maps(pl->e1.p, pl->e1.plane, n, h->conv1_bwd_tc_wt, 80 * 128, err, sizeof(err));
    if (!pl->conv1_bwd_maps) return fail(h, IAN_ERR_CUDA, "enc_conv1_bwd: %s", err);
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  pl->evjp = true;
  return IAN_OK;
}

// the forward (run_encode) on x, then the backward chain.  dz (n,100) is the cotangent of what ian_encode_* returns, taken
// through the MADE/IAF flow's adjoint first; with pre, it is the cotangent of l_Z_IAF (ian_encode_pre_vjp_*) and the chain
// starts at the encoder's sample step.
int run_encode_vjp(ian_handle* h, Plan* pl, const float* x, const float* eps, const float* dz, float* dx, cudaStream_t st,
                   bool pre = false) {
  const int n = pl->n;
  int rc;
  if ((rc = run_encode(h, pl, x, eps, nullptr, st)) != IAN_OK) return rc;
  const float* dzi = dz;
  if (has_flow(h) && !pre) {
    LAUNCH_TRY(h, launch_made_iaf_bwd(pl->z0, h->made_w, h->made_b, dz, pl->edzi, n, st));
    dzi = pl->edzi;
  }
  LAUNCH_TRY(h, launch_enc_vjp_seed(pl->head, eps, dzi, h->w[L_ENC_HEAD].scale, pl->eh.p, pl->eh.plane, n, st));
  for (int l : kEncoderBwd) {
    if ((rc = run_gemm(h, pl, l, st)) != IAN_OK) return rc;
    if (l == E_BWD_HEAD)   // enc_fc1's ReLU / ELU derivative between the head's adjoint and enc_fc1's
      LAUNCH_TRY(h, launch_enc_fc1_bwd(pl->eg, pl->f1.p, pl->f1.plane, h->w[L_ENC_FC1].scale, has_flow(h) ? 0 : 1, pl->ef1.p,
                                       pl->ef1.plane, n, st));
  }
  ScopedTimer tm(h, T_CONV1_BWD, st);
  if (h->path == IAN_PATH_TC)
    LAUNCH_TRY(h, launch_conv1_bwd_tc(pl->conv1_bwd_maps, dx, n, st));
  else
    LAUNCH_TRY(h, launch_conv1_bwd(pl->e1.p, pl->e1.plane, h->conv1_bwd_wt, dx, n, st));
  return IAN_OK;
}

// ---- decoder parameter VJP (IAN_simple) ----------------------------------------------------------------
// dL/dtheta for the 13 trainable decoder tensors of train_IAN_simple.py:353 (`decoder_params`) on the deterministic graph
// of X_hat_fn (API.py:46): inference BatchNorm with mean / inv_std constant.  The chain is the decoder VJP's (run_grad_core
// with the dense seed), so dz is bit for bit ian_decode_vjp_*'s; on top of it:
//   * the forward layers keep their raw pre-BN sums x (out_raw) and the backward-data layers keep their accumulators before
//     mask and scale, which are dL/dh of the layer below (out_raw in ACT_MASK mode); the seed kernel stores dL/dh3 and
//     dec_out's seed image;
//   * weight gradients: the transposes of the four forward tap-GEMMs (wgrad_tc.cu) with G = d0..d3 (dL/d raw output) and
//     A = zp, h0, h1, h2, and dec_out's FFMA reduction (param_vjp.cu);
//   * BatchNorm: d beta = sum dL/dy, d gamma = sum dL/dy * (x - mean) * inv_std, dL/dy = dL/dh * (h > 0) -- no division by
//     gamma or by the folded scale, so a channel with gamma = 0 still gets its gradients.
enum PvSlot { PV_FC2, PV_CONV1, PV_CONV2, PV_CONV3, PV_OUT, PV_BN0_B, PV_BN0_G, PV_BN1_B, PV_BN1_G, PV_BN2_B, PV_BN2_G,
              PV_BN3_B, PV_BN3_G, PV_COUNT };
const char* kPvNames[PV_COUNT] = {"l_dec_fc2.W", "dec_conv1.W", "dec_conv2.W", "dec_conv3.W", "dec_out.W",
                                  "bnorm_dec_fc2.beta", "bnorm_dec_fc2.gamma", "bnorm_dc1.beta", "bnorm_dc1.gamma",
                                  "bnorm_dc2.beta", "bnorm_dc2.gamma", "bnorm_dc3.beta", "bnorm_dc3.gamma"};
const long long kPvSize[PV_COUNT] = {100LL * 16384, 1024LL * 512 * 25, 512LL * 256 * 25, 256LL * 128 * 25, 128LL * 3 * 25,
                                     16384, 16384, 512, 512, 256, 256, 128, 128};
// the split-K slabs of one weight gradient stay within 16 M floats (64 MB per plan: dec_conv1's unsplit slab is 13.1 M)
constexpr long long kWgradMaxWsFloats = 16LL << 20;

int ensure_param_vjp_plan(ian_handle* h, Plan* pl) {
  for (int k = 0; k < 4; ++k)                             // the handle's BN statistics (first call on the handle)
    if (!h->dec_bn_stats[k][0]) {
      int rc = put_dev(h, h->dec_bn_stats[k][0], h->dec_bn[k][2].data(), h->dec_bn[k][2].size() * 4);
      if (rc != IAN_OK) return rc;
      if ((rc = put_dev(h, h->dec_bn_stats[k][1], h->dec_bn[k][3].data(), h->dec_bn[k][3].size() * 4)) != IAN_OK) return rc;
    }
  if (pl->pvjp) return IAN_OK;
  const long long N = pl->n;
  int rc;
#define AP(t, e) if ((rc = alloc_planes(h, pl, pl->t, (e))) != IAN_OK) return rc;
  AP(x0r, N * 16384) AP(x1r, N * 8 * 8 * 512) AP(x2r, N * 16 * 16 * 256) AP(x3r, N * 32 * 32 * 128)
  AP(dh0, N * 16384) AP(dh1, N * 8 * 8 * 512) AP(dh2, N * 16 * 16 * 256) AP(dh3, N * 32 * 32 * 128)
#undef AP
  if ((rc = alloc_buf(h, pl, pl->pseed, N * 3 * 4096)) != IAN_OK) return rc;
  const int* fwd = kSimpleDecoder.fwd.l;
  const Planes* grd[4] = {&pl->d0, &pl->d1, &pl->d2, &pl->d3};
  long long need = 0;
  for (int k = 0; k < 4; ++k) {
    WgradGemm& w = pl->wg[k];
    memset(&w, 0, sizeof(w));
    w.f = pl->g[fwd[k]];
    w.gr = grd[k]->p;
    w.gr_plane = grd[k]->plane;
    w.ws_slab = (long long)h->w[fwd[k]].ntiles * w.f.Cout * w.f.Cin;
    w.ksplit = h->splitk ? wgrad_choose_ksplit(w, kWgradMaxWsFloats) : 1;
    need = std::max(need, w.ksplit * w.ws_slab);
    char err[256] = {0};
    pl->wmaps[k] = wgrad_build_maps(w, err, sizeof(err));
    if (!pl->wmaps[k]) return fail(h, IAN_ERR_CUDA, "wgrad %s: %s", kLayerNames[fwd[k]], err);
  }
  if ((rc = alloc_buf(h, pl, pl->pws, need)) != IAN_OK) return rc;
  for (auto& w : pl->wg) w.ws = pl->pws;
  long long part = (long long)decout_wgrad_chunks(pl->n) * 25 * 384;
  const int bnC[4] = {16384, 512, 256, 128};
  const long long bnR[4] = {N, N * 64, N * 256, N * 1024};
  for (int k = 0; k < 4; ++k) part = std::max(part, (long long)bn_param_chunks(bnC[k], bnR[k]) * 2 * bnC[k]);
  if ((rc = alloc_buf(h, pl, pl->ppart, part)) != IAN_OK) return rc;
  pl->pvjp = true;
  return IAN_OK;
}

// zp holds the latent planes; out[PV_COUNT] device pointers (nullable); accumulate: add into out (a later batch chunk)
int run_param_vjp(ian_handle* h, Plan* pl, const float* dxhat, float* const* out, int accumulate, cudaStream_t st) {
  TapGemm* g = pl->g;
  const int raw_l[7] = {L_DEC_FC2, L_DEC_CONV1, L_DEC_CONV2, L_DEC_CONV3, L_BWD_CONV1, L_BWD_CONV2, L_BWD_CONV3};
  const Planes* raw_p[7] = {&pl->x0r, &pl->x1r, &pl->x2r, &pl->x3r, &pl->dh0, &pl->dh1, &pl->dh2};
  for (int k = 0; k < 7; ++k) { g[raw_l[k]].out_raw = raw_p[k]->p; g[raw_l[k]].out_raw_plane = raw_p[k]->plane; }
  int rc = run_grad_core(h, pl, nullptr, nullptr, 0, dxhat, st, true);
  for (int k = 0; k < 7; ++k) { g[raw_l[k]].out_raw = nullptr; g[raw_l[k]].out_raw_plane = 0; }
  if (rc != IAN_OK) return rc;
  for (int k = 0; k < 4; ++k) {
    if (!out[PV_FC2 + k]) continue;
    {
      ScopedTimer tm(h, T_WGRAD_FC2 + k, st);
      if (h->path == IAN_PATH_TC) LAUNCH_TRY(h, launch_wgrad_tc(pl->wg[k], pl->wmaps[k], st));
      else LAUNCH_TRY(h, launch_wgrad_simt(pl->wg[k], st));
    }
    LAUNCH_TRY(h, launch_wgrad_finalize(pl->wg[k], k == 0 ? WG_FC2 : WG_DECONV, out[PV_FC2 + k], accumulate, st));
  }
  if (out[PV_OUT]) {
    ScopedTimer tm(h, T_WGRAD_DEC_OUT, st);
    LAUNCH_TRY(h, launch_decout_wgrad(pl->pseed, pl->h3.p, pl->h3.plane, pl->n, pl->ppart, out[PV_OUT], accumulate, st));
  }
  const long long N = pl->n;
  struct Bn { const Planes *dh, *hh, *x; int C; long long R; } bns[4] = {
      {&pl->dh0, &pl->h0, &pl->x0r, 16384, N}, {&pl->dh1, &pl->h1, &pl->x1r, 512, N * 64},
      {&pl->dh2, &pl->h2, &pl->x2r, 256, N * 256}, {&pl->dh3, &pl->h3, &pl->x3r, 128, N * 1024}};
  for (int k = 0; k < 4; ++k) {
    float* db = out[PV_BN0_B + 2 * k];
    float* dg = out[PV_BN0_G + 2 * k];
    if (!db && !dg) continue;
    const Bn& b = bns[k];
    LAUNCH_TRY(h, launch_bn_param_bwd(b.dh->p, b.dh->plane, b.hh->p, b.x->p, b.x->plane, h->dec_bn_stats[k][0],
                                      h->dec_bn_stats[k][1], b.C, b.R, k == 0 ? 1 : 0, pl->ppart, db, dg, accumulate, st));
  }
  return IAN_OK;
}

// slot of parameter `index` of ian_model_param_spec, or -1 when the parameter VJP does not compute it
int pv_slot(int model_kind, int index) {
  if (model_kind != IAN_MODEL_SIMPLE) return -1;
  const std::vector<Spec>& specs = cached_specs(IAN_MODEL_SIMPLE);
  if (index < 0 || index >= (int)specs.size()) return -1;
  for (int k = 0; k < PV_COUNT; ++k)
    if (specs[index].name == kPvNames[k]) return k;
  return -1;
}

// common checks; fills out[PV_COUNT] from grads (spec-indexed)
int check_param_vjp(ian_handle* h, const float* z, const float* dx_hat, int n, float* const* grads, float** out) {
  if (!h) return IAN_ERR_INVALID;
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "ian_finalize() has not been called");
  if (h->model_kind != IAN_MODEL_SIMPLE)
    return fail(h, IAN_ERR_UNSUPPORTED, "parameter gradients are implemented for IAN_simple only");
  if (n < 0) return fail(h, IAN_ERR_INVALID, "batch size must not be negative (got %d)", n);
  if (n > 0 && (!z || !dx_hat)) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  for (int k = 0; k < PV_COUNT; ++k) out[k] = nullptr;
  if (!grads) return IAN_OK;
  const std::vector<Spec>& specs = cached_specs(IAN_MODEL_SIMPLE);
  for (int i = 0; i < (int)specs.size(); ++i) {
    if (!grads[i]) continue;
    const int k = pv_slot(h->model_kind, i);
    if (k < 0) return fail(h, IAN_ERR_INVALID, "no gradient is computed for parameter %d ('%s')", i, specs[i].name.c_str());
    out[k] = grads[i];
  }
  return IAN_OK;
}

// the host form's set-up of a plan: the handle's gradient buffers (first call), then the plan's
int prepare_param_vjp_host(ian_handle* h, Plan* pl) {
  for (int k = 0; k < PV_COUNT; ++k)
    if (!h->pv_dev[k]) CUDA_TRY(h, cudaMalloc((void**)&h->pv_dev[k], (size_t)kPvSize[k] * 4));
  return ensure_param_vjp_plan(h, pl);
}

// name and shape of a parameter against the model's list; *elems: its element count
int check_param_shape(ian_handle* h, const char* name, const int64_t* shape, int ndim, int64_t* elems) {
  const Spec* spec = nullptr;
  for (const auto& sp : cached_specs(h->model_kind))
    if (sp.name == name) spec = &sp;
  if (!spec) return fail(h, IAN_ERR_INVALID, "unknown parameter name '%s'", name);
  if (ndim != (int)spec->shape.size()) return fail(h, IAN_ERR_INVALID, "parameter %s: expected %d dims, got %d", name, (int)spec->shape.size(), ndim);
  *elems = 1;
  for (int i = 0; i < ndim; ++i) {
    if (shape[i] != spec->shape[i])
      return fail(h, IAN_ERR_INVALID, "parameter %s: shape mismatch at dim %d (expected %lld, got %lld)", name, i,
                  (long long)spec->shape[i], (long long)shape[i]);
    *elems *= shape[i];
  }
  return IAN_OK;
}

// ---- decoder Jacobian-vector product ----------------------------------------------------------------
// dx_hat = (d x_hat / d z) . v, forward mode through the decoder from l_Z.  A forward layer out = act(BN(conv(in) [+ res]))
// has the tangent t_out = conv(t_in) [+ t_res]) * scale * act'(stored out): the same tap-GEMM (B tiles, taps, geometry, folded
// BatchNorm scale, no shift) on the tangent planes, in ACT_MASK mode with the forward activation as the mask -- the masks and
// scales the decoder VJP applies, so the JVP is the exact transpose of its linear map.  A layer with no activation (IANv1's
// l_dec_fc2) stays ACT_NONE with no shift.  IAN.py's MDBLOCK: the deconv's tangent keeps its raw sum (out_raw), which joins
// MDCL 2's tangent before scale and mask (res, res_after = 0), as in the forward.

// forward plane -> its tangent (a twin's input, residual and mask pointers are looked up here)
using TangentMap = std::map<const void*, const Planes*>;

// Slot lt becomes the tangent twin of forward layer lf (rule above, shared by the decoder and the encoder JVP).  Allocates
// the twin's output planes `out` (and `raw` where the forward keeps its raw sum) and records them in `tan`.
int tangent_twin(ian_handle* h, Plan* pl, int lf, int lt, TangentMap& tan, Planes& out, Planes& raw) {
  const TapGemm& f = pl->g[lf];
  TapGemm& t = pl->g[lt];
  int rc;
  if ((rc = alloc_planes(h, pl, out, f.out_plane)) != IAN_OK) return rc;
  if (f.out_raw && (rc = alloc_planes(h, pl, raw, f.out_raw_plane)) != IAN_OK) return rc;
  if (!tan.count(f.a) || (f.res && !tan.count(f.res)) || (f.act != ACT_NONE && f.act != ACT_RELU && f.act != ACT_LRELU))
    return fail(h, IAN_ERR_STATE, "layer %s: no tangent rule", kLayerNames[lf]);
  t = f;
  t.a = tan[f.a]->p; t.a_plane = tan[f.a]->plane;
  t.shift = nullptr;
  if (f.act != ACT_NONE) { t.act = ACT_MASK; t.mask = f.out; t.mask_slope = f.act == ACT_LRELU ? 0.2f : 0.f; }
  t.out = out.p; t.out_plane = out.plane;
  t.out_raw = f.out_raw ? raw.p : nullptr; t.out_raw_plane = f.out_raw ? raw.plane : 0;
  if (f.res) { t.res = tan[f.res]->p; t.res_plane = tan[f.res]->plane; t.res_after = 0; }
  t.ksplit = 1; t.ws = nullptr;                           // finish_maps decides again, as it did for the forward
  tan[f.out] = &out;
  if (f.out_raw) tan[f.out_raw] = &raw;
  return IAN_OK;
}

// The first call on a plan allocates the tangent planes (the decoder's activations once more) and builds their maps and
// split-K slabs, before any graph capture; plans that never call it keep their memory.
int ensure_jvp_plan(ian_handle* h, Plan* pl) {
  if (pl->jvp) return IAN_OK;
  const DecoderLayers& dec = decoder_layers(h);
  TapGemm* g = pl->g;
  int rc;
  if ((rc = alloc_planes(h, pl, pl->jzp, pl->zp.plane)) != IAN_OK) return rc;
  TangentMap tan = {{pl->zp.p, &pl->jzp}};
  for (int k = 0; k < dec.fwd.n; ++k)
    if ((rc = tangent_twin(h, pl, dec.fwd.l[k], dec.jvp.l[k], tan, pl->jt[k], pl->jr[k])) != IAN_OK) return rc;
  const Planes* t4 = tan[has_flow(h) ? (const void*)pl->fh4.p : (const void*)pl->h3.p];
  LayerList head = {0, {}};
  if (has_flow(h)) {
    g[J_HEAD] = g[F_HEAD];
    g[J_HEAD].a = t4->p; g[J_HEAD].a_plane = t4->plane;   // writes the tap table tt, as the primal head does
    g[J_HEAD].ksplit = 1; g[J_HEAD].ws = nullptr;
    head = {1, {J_HEAD}};
    if ((rc = alloc_buf(h, pl, pl->jrg, (long long)pl->n * 4096 * 4)) != IAN_OK) return rc;
  }
  if ((rc = finish_maps(h, pl, dec.jvp + head)) != IAN_OK) return rc;
  char err[256] = {0};                                    // both paths: ian_set_path may switch a live handle
  if (has_flow(h)) {
    pl->jhead_maps = head_build_maps(t4->p, t4->plane, pl->n, h->head_tc_wt, 3 * 80 * 128, err, sizeof(err));
    if (!pl->jhead_maps) return fail(h, IAN_ERR_CUDA, "rgb head (jvp): %s", err);
  } else {
    pl->jdecout_maps = decout_build_maps(t4->p, t4->plane, pl->n, h->decout_tc_wt, 80 * 128, err, sizeof(err));
    if (!pl->jdecout_maps) return fail(h, IAN_ERR_CUDA, "dec_out (jvp): %s", err);
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  pl->jvp = true;
  return IAN_OK;
}

// the primal (run_decode: the same kernels, so the same x_hat bits and stored activations), then the tangent chain from v
int run_decode_jvp(ian_handle* h, Plan* pl, const float* z, const float* v, float* xhat, float* dxhat, cudaStream_t st) {
  const int n = pl->n;
  int rc;
  if ((rc = run_decode(h, pl, z, xhat, st)) != IAN_OK) return rc;
  LAUNCH_TRY(h, launch_z_to_planes(v, pl->jzp.p, pl->jzp.plane, n, st));
  const DecoderLayers& dec = decoder_layers(h);
  for (int l : dec.jvp)
    if ((rc = run_gemm(h, pl, l, st)) != IAN_OK) return rc;
  const Planes& t4 = pl->jt[dec.jvp.n - 1];
  if (has_flow(h)) {
    if (h->path == IAN_PATH_TC) {
      ScopedTimer tm(h, J_HEAD, st);
      LAUNCH_TRY(h, launch_head_tc(pl->jhead_maps, h->passes, pl->ha, n, st));
    } else {
      if ((rc = run_gemm(h, pl, J_HEAD, st)) != IAN_OK) return rc;
      LAUNCH_TRY(h, launch_head_gather(pl->tt, h->passes == 1 ? 1 : 0, h->head_taps, h->head_ntaps, pl->ha, n, st));
    }
    LAUNCH_TRY(h, launch_rgb_beta_head_jvp(pl->ha, h->path == IAN_PATH_TC ? 1 : 0, pl->rg, pl->bsave, pl->jrg, h->head_taps,
                                           h->head_wgb, h->head_wbb, h->head_ntaps, dxhat, n, st));
    return IAN_OK;
  }
  ScopedTimer tm(h, T_DEC_OUT_JVP, st);
  if (h->path == IAN_PATH_TC)
    LAUNCH_TRY(h, launch_dec_out_jvp_tc(pl->jdecout_maps, xhat, dxhat, n, st));
  else
    LAUNCH_TRY(h, launch_dec_out_jvp(t4.p, t4.plane, h->decout_wt, xhat, dxhat, n, st));
  return IAN_OK;
}

// ---- encoder Jacobian-vector product ----------------------------------------------------------------
// dz = (dz/dx) . v, forward mode through the encoder and, on IAN.py / IANv1.py, the MADE/IAF flow.  With the encoder VJP's
// derivative conventions, so it is the exact transpose of that linear map:
//   enc_conv1: t_a1 = conv1(v) (no bias) * lrelu'(a1), conv1_tc's GEMM (or conv1_kernel's FFMA body) with a mask epilogue;
//   enc_conv2..4: tangent twins (tangent_twin) against a2..a4;
//   enc_fc1: its twin writes float32 with no scale and no activation, then enc_fc1_bwd_kernel -- the encoder VJP's
//            element-wise step -- applies scale * act'(f1) (rectify on the flow graphs, elu' = f1 + 1 on IAN_simple);
//   enc_head: its twin with scale and no shift, float32 [t_mu | t_ls];
//   sample: t_z_iaf = t_mu (+ exp(logsigma) eps t_ls); eps is a constant input;
//   flow: made_iaf_tangent_kernel from the forward's z0.
// enc_conv1 and its tangent run in float32 in either precision, as in the forward.  The first call on a plan allocates the
// tangent planes (the encoder's activations once more, about 1 MB per image) and builds their maps and split-K slabs, before
// any graph capture; plans that never call it keep their memory.
int ensure_enc_jvp_plan(ian_handle* h, Plan* pl) {
  if (pl->ejvp) return IAN_OK;
  const long long N = pl->n;
  TapGemm* g = pl->g;
  int rc;
  if ((rc = alloc_planes(h, pl, pl->jea[0], pl->a1.plane)) != IAN_OK) return rc;
  TangentMap tan = {{pl->a1.p, &pl->jea[0]}};
  Planes raw;                                             // the encoder keeps no raw sums
  for (int k = 0; k < 3; ++k)
    if ((rc = tangent_twin(h, pl, kEncoder.l[k], kEncoderJvp.l[k], tan, pl->jea[k + 1], raw)) != IAN_OK) return rc;
  if ((rc = alloc_planes(h, pl, pl->jef1, pl->f1.plane)) != IAN_OK) return rc;
  if ((rc = alloc_buf(h, pl, pl->jeg, N * 1024)) != IAN_OK) return rc;
  if ((rc = alloc_buf(h, pl, pl->jeh, N * 256)) != IAN_OK) return rc;
  if (has_flow(h) && (rc = alloc_buf(h, pl, pl->jez0, N * 100)) != IAN_OK) return rc;
  TapGemm& fc1 = g[JE_ENC_FC1];
  fc1 = g[L_ENC_FC1];
  fc1.a = pl->jea[3].p; fc1.a_plane = pl->jea[3].plane;
  fc1.act = ACT_NONE; fc1.scale = nullptr; fc1.shift = nullptr;
  fc1.out = nullptr; fc1.out_plane = 0; fc1.out_f32 = pl->jeg;
  fc1.ksplit = 0; fc1.ws = nullptr;                       // as wired for the forward: finish_maps chooses
  TapGemm& head = g[JE_ENC_HEAD];
  head = g[L_ENC_HEAD];
  head.a = pl->jef1.p; head.a_plane = pl->jef1.plane;
  head.shift = nullptr; head.out_f32 = pl->jeh;
  head.ksplit = 1; head.ws = nullptr;
  // the chain's own split-K slabs: the plan's other layers keep theirs
  if ((rc = finish_maps(h, pl, kEncoderJvp)) != IAN_OK) return rc;
  {   // both paths: ian_set_path may switch a live handle
    char err[256] = {0};
    pl->jconv1_out = conv1_build_out_map(pl->jea[0].p, pl->jea[0].plane, pl->n, err, sizeof(err));
    if (!pl->jconv1_out) return fail(h, IAN_ERR_CUDA, "enc_conv1 (jvp): %s", err);
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  pl->ejvp = true;
  return IAN_OK;
}

// the primal (run_encode: the same kernels, so z and the stored activations carry ian_encode_*'s bits), then the tangent chain.
// With pre the chain stops at l_Z_IAF (ian_encode_pre_jvp_*): z (nullable) receives l_Z_IAF as ian_encode_pre_* computes it,
// and dz its tangent, without the flow's.
int run_encode_jvp(ian_handle* h, Plan* pl, const float* x, const float* v, const float* eps, float* z, float* dz, cudaStream_t st,
                   bool pre = false) {
  const int n = pl->n;
  int rc;
  if ((rc = pre ? run_encode(h, pl, x, eps, pl->z, st, z) : run_encode(h, pl, x, eps, z, st)) != IAN_OK) return rc;
  {
    ScopedTimer tm(h, T_CONV1_TANGENT, st);
    if (h->path == IAN_PATH_TC)
      LAUNCH_TRY(h, launch_conv1_tangent_tc(h->conv1_maps, pl->jconv1_out, v, pl->a1.p, n, st));
    else
      LAUNCH_TRY(h, launch_conv1_tangent(v, h->conv1_wt, pl->a1.p, pl->jea[0].p, pl->jea[0].plane, n, st));
  }
  for (int l : kEncoderJvp) {
    if ((rc = run_gemm(h, pl, l, st)) != IAN_OK) return rc;
    if (l == JE_ENC_FC1)   // enc_fc1's BatchNorm scale and ReLU / ELU derivative between its twin and the head's
      LAUNCH_TRY(h, launch_enc_fc1_bwd(pl->jeg, pl->f1.p, pl->f1.plane, h->w[L_ENC_FC1].scale, has_flow(h) ? 0 : 1, pl->jef1.p,
                                       pl->jef1.plane, n, st));
  }
  if (!has_flow(h) || pre) {
    LAUNCH_TRY(h, launch_sample_tangent(pl->head, eps, pl->jeh, dz, n, st));
    return IAN_OK;
  }
  LAUNCH_TRY(h, launch_sample_tangent(pl->head, eps, pl->jeh, pl->jez0, n, st));
  LAUNCH_TRY(h, launch_made_iaf_tangent(pl->z0, pl->jez0, h->made_w, h->made_b, dz, n, st));
  return IAN_OK;
}

// ---- the two forms of an entry point --------------------------------------------------------------
// Each batch entry point is one body over one chunk's device pointers, which run_entry runs in two forms:
//   device form (ian_*_dev): the body on the caller's pointers, offset by the chunk, on the caller's stream;
//   host form (ian_*_host): per chunk, the caller's inputs are copied into plan buffers, the body runs on those, its kernel
//   chain (Chunk::graphed) replayed as a CUDA graph on small plans, the outputs are copied back; then one synchronise.
enum StageBuf { S_X, S_EPS, S_Z, S_XHAT, S_BOXES, S_TARGET, S_EDZ, S_GN_A, S_GN_G, S_GN_E, S_SCALE, S_F1, S_T1 = S_F1 + 4 };
constexpr long long kFeatOff[4] = {0, 131072, 196608, 229376};   // layer l's offset in a sample's 245760 features
void* stage_buf(Plan* pl, int s) {
  if (s >= S_F1) return pl->ifeat + (long long)pl->n * ((s >= S_T1 ? kFeatTotal : 0) + kFeatOff[(s - S_F1) % 4]);
  switch (s) {
    case S_X: return pl->x;
    case S_EPS: return pl->eps;
    case S_Z: return pl->z;
    case S_XHAT: return pl->xhat;
    case S_BOXES: return pl->boxes;
    case S_TARGET: return pl->target;
    case S_GN_A: return pl->gnA;
    case S_GN_G: return pl->gng;
    case S_GN_E: return pl->gne;
    case S_SCALE: return pl->rdl;
    default: return pl->edz;
  }
}
enum { IN = 1, OUT = 2, INOUT = 3 };
struct Arg {              // one per-sample tensor of an entry point
  const void* user;       // the caller's pointer; nullptr: an optional tensor left out
  size_t bytes;           // per sample
  int stage;              // StageBuf: its plan buffer in the host form
  int dir;                // IN, OUT or INOUT
};

struct Chunk {
  ian_handle* h;
  Plan* pl;
  int off, cn;
  cudaStream_t st;
  bool host;
  void* p[10];            // the Args' pointers for this chunk, in order (nullptr for an input left out)
  float* f(int i) const { return (float*)p[i]; }
  const int32_t* i32(int i) const { return (const int32_t*)p[i]; }
  // a kernel chain: replayed from graph `slot` by the host form (run_graphed), launched as is by the device form
  template <typename F>
  int graphed(int slot, uint64_t key, F&& chain) const { return host ? run_graphed(h, pl, slot, key, st, chain) : chain(); }
};

// prepare (nullable): per-plan set-up, run before any staging copy because no allocation may happen during a capture
template <typename Body>
int run_entry(ian_handle* h, bool host, void* stream, int n, std::initializer_list<Arg> args, int (*prepare)(ian_handle*, Plan*),
              Body&& body) {
  DeviceGuard dg(h->device);
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  const int rc = for_chunks(h, n, [&](Plan* pl, int off, int cn) {
    int r = prepare ? prepare(h, pl) : (int)IAN_OK;
    if (r != IAN_OK) return r;
    Chunk c{h, pl, off, cn, st, host, {}};
    int i = 0;
    for (const Arg& a : args) {
      char* u = a.user ? (char*)a.user + (size_t)off * a.bytes : nullptr;
      void* p = !host ? u : (u || a.dir != IN) ? stage_buf(pl, a.stage) : nullptr;
      if (host && u && (a.dir & IN)) CUDA_TRY(h, cudaMemcpyAsync(p, u, (size_t)cn * a.bytes, cudaMemcpyHostToDevice, st));
      c.p[i++] = p;
    }
    if ((r = body(c)) != IAN_OK) return r;
    i = 0;
    for (const Arg& a : args) {
      void* p = c.p[i++];
      if (host && a.user && (a.dir & OUT))
        CUDA_TRY(h, cudaMemcpyAsync((char*)a.user + (size_t)off * a.bytes, p, (size_t)cn * a.bytes, cudaMemcpyDeviceToHost, st));
    }
    return (int)IAN_OK;
  });
  if (rc != IAN_OK || !host) return rc;
  CUDA_TRY(h, cudaStreamSynchronize(st));
  return IAN_OK;
}

constexpr size_t kImageBytes = 12288 * 4, kLatentBytes = 400;

// dz: columns 0..99 of gpad (n,128), a pitched copy (no box, so no empty-box NaN rule)
int copy_dz(const Chunk& c, float* dz) {
  if (dz)
    CUDA_TRY(c.h, cudaMemcpy2DAsync(dz + (size_t)c.off * 100, 400, c.pl->gpad, 512, 400, c.cn,
                                    c.host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c.st));
  return IAN_OK;
}

int call_encode(ian_handle* h, bool host, const float* x, int n, const float* eps, float* z, void* stream) {
  int rc = check_ready(h, n, x, z);
  if (rc != IAN_OK) return rc;
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {eps, kLatentBytes, S_EPS, IN}, {z, kLatentBytes, S_Z, OUT}},
                   nullptr, [&](const Chunk& c) {
    return c.graphed(eps ? Plan::G_ENCODE_EPS : Plan::G_ENCODE, 0,
                     [&] { return run_encode(h, c.pl, c.f(0), c.f(1), c.f(2), c.st); });
  });
}

int call_decode(ian_handle* h, bool host, const float* z, int n, float* x, void* stream) {
  int rc = check_ready(h, n, z, x);
  if (rc != IAN_OK) return rc;
  return run_entry(h, host, stream, n, {{z, kLatentBytes, S_Z, IN}, {x, kImageBytes, S_XHAT, OUT}}, nullptr,
                   [&](const Chunk& c) {
    return c.graphed(Plan::G_DECODE, 0, [&] { return run_decode(h, c.pl, c.f(0), c.f(1), c.st); });
  });
}

int call_reconstruct(ian_handle* h, bool host, const float* x, int n, float* z_out, float* x_hat, void* stream) {
  int rc = check_ready(h, n, x, x_hat);
  if (rc != IAN_OK) return rc;
  return run_entry(h, host, stream, n,
                   {{x, kImageBytes, S_X, IN}, {z_out, kLatentBytes, S_Z, OUT}, {x_hat, kImageBytes, S_XHAT, OUT}}, nullptr,
                   [&](const Chunk& c) {
    return c.graphed(Plan::G_RECON, 0, [&] {
      int q = run_encode(h, c.pl, c.f(0), nullptr, c.f(1), c.st);
      return q != IAN_OK ? q : run_decode_from_planes(h, c.pl, c.f(2), c.st);
    });
  });
}

int call_grad(ian_handle* h, bool host, const float* z, const int32_t* boxes, const float* target, int target_is_frame, int n,
              float* g, void* stream) {
  int rc = check_ready(h, n, z, g);
  if (rc != IAN_OK) return rc;
  if (!boxes) return fail(h, IAN_ERR_INVALID, "boxes is NULL");
  if (host && (rc = validate_boxes(h, boxes, n)) != IAN_OK) return rc;
  const size_t tbytes = (target_is_frame ? 12288 : 3) * 4;
  // the host form stages g in z's buffer
  return run_entry(h, host, stream, n, {{z, kLatentBytes, S_Z, IN}, {boxes, 16, S_BOXES, IN}, {target, tbytes, S_TARGET, IN},
                                        {g, kLatentBytes, S_Z, OUT}}, nullptr, [&](const Chunk& c) {
    return c.graphed(Plan::G_GRAD, (target ? 1 : 0) + (target_is_frame ? 2 : 0), [&] {
      LAUNCH_TRY(h, launch_z_to_planes(c.f(0), c.pl->zp.p, c.pl->zp.plane, c.cn, c.st));
      int q = run_grad_core(h, c.pl, c.i32(1), c.f(2), target_is_frame, nullptr, c.st);
      if (q != IAN_OK) return q;
      LAUNCH_TRY(h, launch_brush_update(c.pl->gpad, c.i32(1), 0.f, c.f(3), nullptr, nullptr, 0, c.cn, c.st));
      return (int)IAN_OK;
    });
  });
}

// The brush gradient's kernels with the dense seed (run_grad_core, dxhat set); the host form stages the cotangent in the
// plan's frame-target buffer (n,3,64,64).
int call_decode_vjp(ian_handle* h, bool host, const float* z, const float* dx_hat, int n, float* dz, void* stream) {
  int rc = check_ready(h, n, z, dz);
  if (rc != IAN_OK) return rc;
  if (!dx_hat) return fail(h, IAN_ERR_INVALID, "dx_hat is NULL");
  return run_entry(h, host, stream, n, {{z, kLatentBytes, S_Z, IN}, {dx_hat, kImageBytes, S_TARGET, IN}}, nullptr,
                   [&](const Chunk& c) {
    int r = c.graphed(Plan::G_VJP, 0, [&] {
      LAUNCH_TRY(h, launch_z_to_planes(c.f(0), c.pl->zp.p, c.pl->zp.plane, c.cn, c.st));
      return run_grad_core(h, c.pl, nullptr, nullptr, 0, c.f(1), c.st);
    });
    return r != IAN_OK ? r : copy_dz(c, dz);
  });
}

// The host form computes every gradient into the handle's device buffers (allocated on the first call), so a captured graph
// does not depend on which ones the caller asked for; the requested ones are copied out after the last chunk.
int call_param_vjp(ian_handle* h, bool host, const float* z, const float* dx_hat, int n, float* dz, float* const* grads,
                   void* stream) {
  float* req[PV_COUNT];
  int rc = check_param_vjp(h, z, dx_hat, n, grads, req);
  if (rc != IAN_OK || n == 0) return rc;
  return run_entry(h, host, stream, n, {{z, kLatentBytes, S_Z, IN}, {dx_hat, kImageBytes, S_TARGET, IN}},
                   host ? prepare_param_vjp_host : ensure_param_vjp_plan, [&](const Chunk& c) {
    const int accumulate = c.off > 0;
    int r = c.graphed(Plan::G_PARAM_VJP, accumulate, [&] {
      LAUNCH_TRY(h, launch_z_to_planes(c.f(0), c.pl->zp.p, c.pl->zp.plane, c.cn, c.st));
      return run_param_vjp(h, c.pl, c.f(1), host ? h->pv_dev : req, accumulate, c.st);
    });
    if (r == IAN_OK) r = copy_dz(c, dz);
    if (r != IAN_OK || !host || c.off + c.cn < n) return r;
    for (int k = 0; k < PV_COUNT; ++k)
      if (req[k]) CUDA_TRY(h, cudaMemcpyAsync(req[k], h->pv_dev[k], (size_t)kPvSize[k] * 4, cudaMemcpyDeviceToHost, c.st));
    return (int)IAN_OK;
  });
}

// The first call on a handle permutes the backward weight tiles; the first call on a plan allocates its gradient planes
// and tensor maps (about 1 MB per image).  Both happen before any graph capture; handles and plans that never call these
// keep their memory as it was.  The host form stages dz in the plan's edz buffer and dx in its x_hat buffer.
int call_encode_vjp(ian_handle* h, bool host, const float* x, int n, const float* eps, const float* dz, float* dx, void* stream) {
  int rc = check_ready(h, n, x, dx);
  if (rc != IAN_OK) return rc;
  if (!dz) return fail(h, IAN_ERR_INVALID, "dz is NULL");
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {eps, kLatentBytes, S_EPS, IN}, {dz, kLatentBytes, S_EDZ, IN},
                                        {dx, kImageBytes, S_XHAT, OUT}}, ensure_enc_vjp_plan, [&](const Chunk& c) {
    return c.graphed(Plan::G_ENC_VJP, eps ? 1 : 0,
                     [&] { return run_encode_vjp(h, c.pl, c.f(0), c.f(1), c.f(2), c.f(3), c.st); });
  });
}

// x_hat is nullable: the primal then goes to the plan's x_hat buffer.  The host form stages v in the plan's eps buffer,
// x_hat in its x_hat buffer and dx_hat in its image buffer.
int call_decode_jvp(ian_handle* h, bool host, const float* z, const float* v, int n, float* x_hat, float* dx_hat, void* stream) {
  if (!h) return IAN_ERR_INVALID;
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "ian_finalize() has not been called");
  if (n < 0) return fail(h, IAN_ERR_INVALID, "batch size must not be negative (got %d)", n);
  if (n == 0) return IAN_OK;
  if (!z || !v || !dx_hat) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  return run_entry(h, host, stream, n, {{z, kLatentBytes, S_Z, IN}, {v, kLatentBytes, S_EPS, IN}, {x_hat, kImageBytes, S_XHAT, OUT},
                                        {dx_hat, kImageBytes, S_X, OUT}}, ensure_jvp_plan, [&](const Chunk& c) {
    return c.graphed(Plan::G_JVP, 0, [&] {
      return run_decode_jvp(h, c.pl, c.f(0), c.f(1), c.f(2) ? c.f(2) : c.pl->xhat, c.f(3), c.st);
    });
  });
}

// z is nullable: the primal then goes to the plan's z buffer.  The host form stages v in the plan's frame-target buffer,
// z in its z buffer and dz in its x_hat buffer.
int call_encode_jvp(ian_handle* h, bool host, const float* x, const float* v, int n, const float* eps, float* z, float* dz,
                    void* stream) {
  if (!h) return IAN_ERR_INVALID;
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "ian_finalize() has not been called");
  if (n < 0) return fail(h, IAN_ERR_INVALID, "batch size must not be negative (got %d)", n);
  if (n == 0) return IAN_OK;
  if (!x || !v || !dz) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {v, kImageBytes, S_TARGET, IN}, {eps, kLatentBytes, S_EPS, IN},
                                        {z, kLatentBytes, S_Z, OUT}, {dz, kLatentBytes, S_XHAT, OUT}}, ensure_enc_jvp_plan,
                   [&](const Chunk& c) {
    return c.graphed(Plan::G_ENC_JVP, eps ? 1 : 0, [&] {
      return run_encode_jvp(h, c.pl, c.f(0), c.f(1), c.f(2), c.f(3) ? c.f(3) : c.pl->z, c.f(4), c.st);
    });
  });
}

// ---- the sampling script's function set and its derivatives (sample_IAN.py:86-94) ----------------------------------------
// Zfn: X -> l_Z_IAF (deterministic: mu).  The encoder's kernels with l_Z_IAF kept (run_encode's z_pre); the host form stages
// it in the plan's eps buffer.
int call_encode_pre(ian_handle* h, bool host, const float* x, int n, float* z_iaf, void* stream) {
  int rc = check_ready(h, n, x, z_iaf);
  if (rc != IAN_OK) return rc;
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {z_iaf, kLatentBytes, S_EPS, OUT}}, nullptr,
                   [&](const Chunk& c) {
    return c.graphed(Plan::G_ENCODE_PRE, 0, [&] { return run_encode(h, c.pl, c.f(0), nullptr, c.pl->z, c.st, c.f(1)); });
  });
}

// z = F(u) as ian_flow_* computes it, with made_iaf_kernel also writing zp when given; a copy of u on IAN_simple
int flow_z(ian_handle* h, const float* u, float* z, Planes* zp, int n, cudaStream_t st) {
  if (has_flow(h)) {
    LAUNCH_TRY(h, launch_made_iaf(u, h->made_w, h->made_b, z, zp ? zp->p : nullptr, zp ? zp->plane : 0, n, st));
    return IAN_OK;
  }
  CUDA_TRY(h, cudaMemcpyAsync(z, u, (size_t)n * 400, cudaMemcpyDeviceToDevice, st));
  return IAN_OK;
}

// l_Z_IAF -> l_Z (Z_IAF_fn) into z_out or the plan's z buffer, and the latent planes; x_out != NULL also decodes them
// (`sample`).  The host form stages z_iaf in the plan's eps buffer; it decides on the caller's pointers, because it stages
// every output whether asked for or not.
int run_flow(ian_handle* h, Plan* pl, const float* z_iaf, float* z, cudaStream_t st) {
  const int rc = flow_z(h, z_iaf, z, &pl->zp, pl->n, st);
  if (rc != IAN_OK || has_flow(h)) return rc;
  LAUNCH_TRY(h, launch_z_to_planes(z, pl->zp.p, pl->zp.plane, pl->n, st));
  return IAN_OK;
}

int call_flow(ian_handle* h, bool host, const float* z_iaf, int n, float* z_out, float* x_out, void* stream) {
  int rc = check_ready(h, n, z_iaf, z_iaf);
  if (rc != IAN_OK) return rc;
  if (!z_out && !x_out) return fail(h, IAN_ERR_INVALID, "both outputs are NULL");
  return run_entry(h, host, stream, n, {{z_iaf, kLatentBytes, S_EPS, IN}, {z_out, kLatentBytes, S_Z, OUT},
                                        {x_out, kImageBytes, S_XHAT, OUT}}, nullptr, [&](const Chunk& c) {
    return c.graphed(Plan::G_FLOW, x_out ? 1 : 0, [&] {
      int q = run_flow(h, c.pl, c.f(0), z_out ? c.f(1) : c.pl->z, c.st);
      return q != IAN_OK || !x_out ? q : run_decode_from_planes(h, c.pl, c.f(2), c.st);
    });
  });
}

int check_flow_grad(ian_handle* h, int n, const void* a, const void* b, const void* c) {
  if (!h) return IAN_ERR_INVALID;
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "ian_finalize() has not been called");
  if (n < 0) return fail(h, IAN_ERR_INVALID, "batch size must not be negative (got %d)", n);
  if (n > 0 && (!a || !b || !c)) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  return IAN_OK;
}

// dz_iaf = (d l_Z / d l_Z_IAF)^T dz: made_iaf_bwd_kernel on the caller's z_iaf (a copy of dz on IAN_simple).  Needs only the
// plan's (n,100) buffers: the host form stages z_iaf in its eps buffer, dz in its frame-target buffer and dz_iaf in its z buffer.
int call_flow_vjp(ian_handle* h, bool host, const float* z_iaf, const float* dz, int n, float* dz_iaf, void* stream) {
  int rc = check_flow_grad(h, n, z_iaf, dz, dz_iaf);
  if (rc != IAN_OK || n == 0) return rc;
  return run_entry(h, host, stream, n, {{z_iaf, kLatentBytes, S_EPS, IN}, {dz, kLatentBytes, S_TARGET, IN},
                                        {dz_iaf, kLatentBytes, S_Z, OUT}}, nullptr, [&](const Chunk& c) {
    return c.graphed(Plan::G_FLOW_VJP, 0, [&] {
      if (has_flow(h))
        LAUNCH_TRY(h, launch_made_iaf_bwd(c.f(0), h->made_w, h->made_b, c.f(1), c.f(2), c.cn, c.st));
      else if (c.f(2) != c.f(1))
        CUDA_TRY(h, cudaMemcpyAsync(c.f(2), c.f(1), (size_t)c.cn * 400, cudaMemcpyDeviceToDevice, c.st));
      return (int)IAN_OK;
    });
  });
}

// dz = (d l_Z / d l_Z_IAF) . v: made_iaf_tangent_kernel on the caller's z_iaf, after made_iaf_kernel for the primal when z is
// wanted (v and z_iaf copied on IAN_simple).  The host form stages z_iaf in the eps buffer, v in the frame-target buffer, z in
// the z buffer and dz in the x_hat buffer.
int call_flow_jvp(ian_handle* h, bool host, const float* z_iaf, const float* v, int n, float* z, float* dz, void* stream) {
  int rc = check_flow_grad(h, n, z_iaf, v, dz);
  if (rc != IAN_OK || n == 0) return rc;
  return run_entry(h, host, stream, n, {{z_iaf, kLatentBytes, S_EPS, IN}, {v, kLatentBytes, S_TARGET, IN},
                                        {z, kLatentBytes, S_Z, OUT}, {dz, kLatentBytes, S_XHAT, OUT}}, nullptr,
                   [&](const Chunk& c) {
    return c.graphed(Plan::G_FLOW_JVP, z ? 1 : 0, [&] {
      const size_t bytes = (size_t)c.cn * 400;
      if (has_flow(h)) {
        if (z) LAUNCH_TRY(h, launch_made_iaf(c.f(0), h->made_w, h->made_b, c.f(2), nullptr, 0, c.cn, c.st));
        LAUNCH_TRY(h, launch_made_iaf_tangent(c.f(0), c.f(1), h->made_w, h->made_b, c.f(3), c.cn, c.st));
        return (int)IAN_OK;
      }
      if (z && c.f(2) != c.f(0)) CUDA_TRY(h, cudaMemcpyAsync(c.f(2), c.f(0), bytes, cudaMemcpyDeviceToDevice, c.st));
      if (c.f(3) != c.f(1)) CUDA_TRY(h, cudaMemcpyAsync(c.f(3), c.f(1), bytes, cudaMemcpyDeviceToDevice, c.st));
      return (int)IAN_OK;
    });
  });
}

// Zfn's VJP: the encoder VJP's chain seeded with dz_iaf at the sample step, eps absent.  The host form stages dz_iaf in the
// plan's edz buffer and dx in its x_hat buffer.
int call_encode_pre_vjp(ian_handle* h, bool host, const float* x, int n, const float* dz_iaf, float* dx, void* stream) {
  int rc = check_flow_grad(h, n, x, dz_iaf, dx);
  if (rc != IAN_OK || n == 0) return rc;
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {dz_iaf, kLatentBytes, S_EDZ, IN},
                                        {dx, kImageBytes, S_XHAT, OUT}}, ensure_enc_vjp_plan, [&](const Chunk& c) {
    return c.graphed(Plan::G_ENC_PRE_VJP, 0,
                     [&] { return run_encode_vjp(h, c.pl, c.f(0), nullptr, c.f(1), c.f(2), c.st, true); });
  });
}

// Zfn's JVP: the encoder JVP's chain up to the tangent of l_Z_IAF, eps absent.  z_iaf is nullable.  The host form stages v in
// the plan's frame-target buffer, z_iaf in its eps buffer and dz_iaf in its x_hat buffer.
int call_encode_pre_jvp(ian_handle* h, bool host, const float* x, const float* v, int n, float* z_iaf, float* dz_iaf,
                        void* stream) {
  int rc = check_flow_grad(h, n, x, v, dz_iaf);
  if (rc != IAN_OK || n == 0) return rc;
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {v, kImageBytes, S_TARGET, IN},
                                        {z_iaf, kLatentBytes, S_EPS, OUT}, {dz_iaf, kLatentBytes, S_XHAT, OUT}},
                   ensure_enc_jvp_plan, [&](const Chunk& c) {
    return c.graphed(Plan::G_ENC_PRE_JVP, 0,
                     [&] { return run_encode_jvp(h, c.pl, c.f(0), c.f(1), nullptr, c.f(2), c.f(3), c.st, true); });
  });
}

// The host form captures one paint step and replays it n_steps times; its key holds the weight's bits.
int call_edit_loop(ian_handle* h, bool host, float* z, const int32_t* boxes, const float* target, int target_is_frame, int n,
                   int n_steps, float weight, void* stream) {
  int rc = check_ready(h, n, z, z);
  if (rc != IAN_OK) return rc;
  if (!boxes) return fail(h, IAN_ERR_INVALID, "boxes is NULL");
  if (!host && n_steps < 0) return fail(h, IAN_ERR_INVALID, "n_steps < 0");
  if (host && (rc = validate_boxes(h, boxes, n)) != IAN_OK) return rc;
  const size_t tbytes = (target_is_frame ? 12288 : 3) * 4;
  const uint64_t key = float_bits(weight) * 4 + (target ? 1 : 0) + (target_is_frame ? 2 : 0);
  return run_entry(h, host, stream, n, {{z, kLatentBytes, S_Z, INOUT}, {boxes, 16, S_BOXES, IN}, {target, tbytes, S_TARGET, IN}},
                   nullptr, [&](const Chunk& c) {
    LAUNCH_TRY(h, launch_z_to_planes(c.f(0), c.pl->zp.p, c.pl->zp.plane, c.cn, c.st));
    for (int s = 0; s < n_steps; ++s) {
      int r = c.graphed(Plan::G_EDIT_STEP, key, [&] {
        int q = run_grad_core(h, c.pl, c.i32(1), c.f(2), target_is_frame, nullptr, c.st);
        if (q != IAN_OK) return q;
        LAUNCH_TRY(h, launch_brush_update(c.pl->gpad, c.i32(1), weight, nullptr, c.f(0), c.pl->zp.p, c.pl->zp.plane, c.cn, c.st));
        return (int)IAN_OK;
      });
      if (r != IAN_OK) return r;
    }
    return (int)IAN_OK;
  });
}

// ---- latent fit: Levenberg-Marquardt on the decoder's Gauss-Newton normal equations (DESIGN section 5.6i) ----------------
// r = x_hat - x comes from run_decode on the caller's batch plan, so x_hat has ian_decode_*'s bits at that batch size.  J
// comes from run_decode_jvp on the 100-row plan that decoder_jacobian uses -- the latent replicated 100 times, the identity
// as tangents -- one sample per pass, so the JVP's memory stays what a batch-100 ian_decode_jvp_* call allocates, plus the
// 4.9 MB J buffer on the handle.  The first call on a handle allocates the handle's buffers and the 100-row plan's tangent
// planes; the first call on a plan its normal equations and fit state (about 180 KB per image); all before any launch.
int ensure_gn_plan(ian_handle* h, Plan* pl) {
  int rc;
  if (!h->gn_part) {
    std::vector<float> eye(10000, 0.f);
    for (int i = 0; i < 100; ++i) eye[i * 101] = 1.f;
    if ((rc = put_dev(h, h->gn_eye, eye.data(), eye.size() * sizeof(float))) != IAN_OK) return rc;
    if (!h->gn_zrep) CUDA_TRY(h, cudaMalloc((void**)&h->gn_zrep, 10000 * sizeof(float)));
    if (!h->gn_J) CUDA_TRY(h, cudaMalloc((void**)&h->gn_J, (size_t)100 * 12288 * sizeof(float)));
    CUDA_TRY(h, cudaMalloc((void**)&h->gn_part, gn_part_doubles() * sizeof(double)));
  }
  Plan* jp = nullptr;
  if ((rc = get_plan(h, 100, &jp)) != IAN_OK || (rc = ensure_jvp_plan(h, jp)) != IAN_OK) return rc;
  if (pl->gn) return IAN_OK;
  const long long N = pl->n;
  if ((rc = alloc_buf(h, pl, pl->gnA, N * 10000)) != IAN_OK || (rc = alloc_buf(h, pl, pl->gng, N * 100)) != IAN_OK ||
      (rc = alloc_buf(h, pl, pl->gne, N)) != IAN_OK || (rc = alloc_buf(h, pl, pl->fe, N)) != IAN_OK ||
      (rc = alloc_buf(h, pl, pl->flam, N)) != IAN_OK || (rc = alloc_buf(h, pl, pl->fxh, N * 12288)) != IAN_OK ||
      (rc = alloc_buf(h, pl, pl->fxt, N * 12288)) != IAN_OK || (rc = alloc_buf(h, pl, pl->fzt, N * 100)) != IAN_OK ||
      (rc = alloc_buf(h, pl, pl->fok, N)) != IAN_OK)
    return rc;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  pl->gn = true;
  return IAN_OK;
}

// the workspace of the training-mode ops and the discriminator head's MinibatchLayer
int ensure_train_ws(ian_handle* h, size_t bytes) {
  if (bytes <= h->train_ws_bytes) return IAN_OK;
  if (h->train_ws) { CUDA_TRY(h, cudaDeviceSynchronize()); CUDA_TRY(h, cudaFree(h->train_ws)); h->train_ws = nullptr; h->train_ws_bytes = 0; }
  CUDA_TRY(h, cudaMalloc(&h->train_ws, bytes));
  h->train_ws_bytes = bytes;
  return IAN_OK;
}

// The first checks of the fit and introspection entries: the handle, n and iters (the fits).  The fits then check their
// objective's own arguments (check_robust_args, check_feat_weights), then n == 0 and the rest (check_fit_inputs).
int check_fit_args(ian_handle* h, int n, int iters = 0) {
  if (!h) return IAN_ERR_INVALID;
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "ian_finalize() has not been called");
  if (n < 0) return fail(h, IAN_ERR_INVALID, "batch size must not be negative (got %d)", n);
  if (iters < 0) return fail(h, IAN_ERR_INVALID, "iters must not be negative (got %d)", iters);
  return IAN_OK;
}

// The fit's loss history (nullable) of one chunk, row stride ldl: the caller's rows in the device form; in the host form a
// plan buffer grown to the largest (chunk, iters) asked for, copied out by fit_loss_out.
int fit_loss_buf(const Chunk& c, float* loss, size_t ldl, float** l) {
  *l = loss && !c.host ? loss + (size_t)c.off * ldl : nullptr;
  const long long need = (long long)(c.cn * ldl);
  if (loss && c.host) {
    if (c.pl->floss_cap < need) {
      CUDA_TRY(c.h, cudaFree(c.pl->floss));
      c.pl->floss = nullptr;
      c.pl->floss_cap = 0;
      CUDA_TRY(c.h, cudaMalloc((void**)&c.pl->floss, (size_t)need * sizeof(float)));
      c.pl->floss_cap = need;
    }
    *l = c.pl->floss;
  }
  return IAN_OK;
}

int fit_loss_out(const Chunk& c, float* loss, size_t ldl, const float* l) {
  if (loss && c.host)
    CUDA_TRY(c.h, cudaMemcpyAsync(loss + (size_t)c.off * ldl, l, c.cn * ldl * sizeof(float), cudaMemcpyDeviceToHost, c.st));
  return IAN_OK;
}

// ---- masked latent fit under the prior: pixel-weighted Levenberg-Marquardt in the fit space u (DESIGN section 5.6j) -------
// u is l_Z on IAN_simple and l_Z_IAF on IAN.py / IANv1.py, and z = F(u) the MADE/IAF flow (the identity on IAN_simple).
// x_hat = decode(F(u)) on the caller's batch plan: made_iaf_kernel writes the latent planes as `sample` does, so x_hat has
// ian_flow_*'s bits with x_out at that batch size (on IAN_simple run_decode, the fit's own).  J_u = J_dec(F(u)) J_F(u)
// comes from one batch-100 pass per sample on the plan the fit uses: u replicated 100 times, the flow's z rows and its
// JVP with the identity as tangents (the kernels of ian_flow_jvp_*), then run_decode_jvp with those rows as tangents.  On
// IAN_simple the pass is the fit's own.  The first call on a handle also allocates the flow's 80 KB of rows (flow graphs).
int ensure_map_plan(ian_handle* h, Plan* pl) {
  int rc = ensure_gn_plan(h, pl);
  if (rc != IAN_OK) return rc;
  if (has_flow(h) && !h->map_flow) CUDA_TRY(h, cudaMalloc((void**)&h->map_flow, 20000 * sizeof(float)));
  return IAN_OK;
}

// ---- robust latent fit: Huber / Cauchy pixel losses by reweighted Levenberg-Marquardt (DESIGN section 5.6m) -------------
// The masked fit's passes, plan and rule with the Gram reweighted by rho' and the accept rule on the true robust E.
static_assert(IAN_ROBUST_HUBER == kRobustHuber && IAN_ROBUST_CAUCHY == kRobustCauchy,
              "the kernels compare the header's loss ids with edge.h's");
int ensure_robust_plan(ian_handle* h, Plan* pl) {
  int rc = ensure_map_plan(h, pl);
  if (rc != IAN_OK || pl->rdl) return rc;
  if ((rc = alloc_buf(h, pl, pl->rdl, pl->n)) != IAN_OK) return rc;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return IAN_OK;
}

// kind, and (host form) every scale: > 0 and not NaN, +inf for Huber only
int check_robust_args(ian_handle* h, bool host, int n, int kind, const double* scale) {
  if (kind != IAN_ROBUST_HUBER && kind != IAN_ROBUST_CAUCHY) return fail(h, IAN_ERR_INVALID, "unknown robust loss kind %d", kind);
  if (host && scale)
    for (int k = 0; k < n; ++k)
      if (!(scale[k] > 0.0) || (std::isinf(scale[k]) && kind == IAN_ROBUST_CAUCHY))
        return fail(h, IAN_ERR_INVALID, "scale %d is %g: scales must be > 0, and finite for the Cauchy loss", k, scale[k]);
  return IAN_OK;
}

// ---- the IAN's introspection features and the fit under its feature-wise loss (DESIGN section 5.6k) --------------------
// g_1..g_4 are the encoder's activations a1..a4 (enc_conv1..4 after BatchNorm and LeakyReLU, inference BatchNorm): the
// encoder forward stopped after enc_conv4, and the feature values are what it stores (hi + lo, or hi in bf16 mode).
const Planes& feat_planes(Plan* pl, int l) { return l == 0 ? pl->a1 : l == 1 ? pl->a2 : l == 2 ? pl->a3 : pl->a4; }

// depth < 4: the forward stops after enc_conv{depth}
int run_introspect(ian_handle* h, Plan* pl, const float* x, cudaStream_t st, int depth = 4) {
  {
    ScopedTimer tm(h, T_CONV1, st);
    if (h->path == IAN_PATH_TC)
      LAUNCH_TRY(h, launch_conv1_tc(h->conv1_maps, pl->conv1_out, x, h->conv1_b, pl->n, st));
    else
      LAUNCH_TRY(h, launch_conv1(x, h->conv1_wt, h->conv1_b, pl->a1.p, pl->a1.plane, pl->n, st));
  }
  int rc;
  for (int k = 0; k < depth - 1; ++k)
    if ((rc = run_gemm(h, pl, kEncoder.l[k], st)) != IAN_OK) return rc;
  return IAN_OK;
}

// run_encode_jvp's tangent chain truncated after jvp_enc_conv4: the tangents of a1..a4 in pl->jea[0..3]
int run_introspect_jvp(ian_handle* h, Plan* pl, const float* x, const float* v, cudaStream_t st) {
  int rc = run_introspect(h, pl, x, st);
  if (rc != IAN_OK) return rc;
  {
    ScopedTimer tm(h, T_CONV1_TANGENT, st);
    if (h->path == IAN_PATH_TC)
      LAUNCH_TRY(h, launch_conv1_tangent_tc(h->conv1_maps, pl->jconv1_out, v, pl->a1.p, pl->n, st));
    else
      LAUNCH_TRY(h, launch_conv1_tangent(v, h->conv1_wt, pl->a1.p, pl->jea[0].p, pl->jea[0].plane, pl->n, st));
  }
  for (int k = 0; k < 3; ++k)
    if ((rc = run_gemm(h, pl, kEncoderJvp.l[k], st)) != IAN_OK) return rc;
  return IAN_OK;
}

// the plan's four feature planes (tangent: their tangents) -> float32: out[l] nullable, NCHW per layer, or NHWC at
// base + n * off_l
int store_features(ian_handle* h, Plan* pl, bool tangent, float* const* out, float* base, int nchw, cudaStream_t st) {
  for (int l = 0; l < 4; ++l) {
    const Planes& src = tangent ? pl->jea[l] : feat_planes(pl, l);
    float* o = base ? base + (long long)pl->n * kFeatOff[l] : out[l];
    if (o) LAUNCH_TRY(h, launch_feat_store(src.p, src.plane, h->passes, l, pl->n, o, nchw, st));
  }
  return IAN_OK;
}

// The host forms stage the outputs in a plan buffer of 1.97 MB per image (features, then tangents), allocated on their
// first call on the plan; the device forms allocate nothing for the features.
template <bool kHost, bool kJvp>
int ensure_introspect_plan(ian_handle* h, Plan* pl) {
  int rc;
  if (kJvp && (rc = ensure_enc_jvp_plan(h, pl)) != IAN_OK) return rc;
  if (kHost && !pl->ifeat) {
    if ((rc = alloc_buf(h, pl, pl->ifeat, (long long)pl->n * 2 * kFeatTotal)) != IAN_OK) return rc;
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  return IAN_OK;
}

constexpr size_t kFeatBytes[4] = {131072 * 4, 65536 * 4, 32768 * 4, 16384 * 4};

// No CUDA graphs: the features are a measurement and a building block, not an interactive call.
int call_introspect(ian_handle* h, bool host, const float* x, int n, float* const* f, void* stream) {
  int rc = check_fit_args(h, n);
  if (rc != IAN_OK || n == 0) return rc;
  if (!x) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {f[0], kFeatBytes[0], S_F1, OUT},
                                        {f[1], kFeatBytes[1], S_F1 + 1, OUT}, {f[2], kFeatBytes[2], S_F1 + 2, OUT},
                                        {f[3], kFeatBytes[3], S_F1 + 3, OUT}},
                   host ? ensure_introspect_plan<true, false> : ensure_introspect_plan<false, false>, [&](const Chunk& c) {
    const int r = run_introspect(h, c.pl, c.f(0), c.st);
    float* o[4] = {c.f(1), c.f(2), c.f(3), c.f(4)};
    return r != IAN_OK ? r : store_features(h, c.pl, false, o, nullptr, 1, c.st);
  });
}

int call_introspect_jvp(ian_handle* h, bool host, const float* x, const float* v, int n, float* const* f, float* const* t,
                        void* stream) {
  int rc = check_fit_args(h, n);
  if (rc != IAN_OK || n == 0) return rc;
  if (!x || !v || !t[0] || !t[1] || !t[2] || !t[3]) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {v, kImageBytes, S_TARGET, IN},
                                        {f[0], kFeatBytes[0], S_F1, OUT}, {f[1], kFeatBytes[1], S_F1 + 1, OUT},
                                        {f[2], kFeatBytes[2], S_F1 + 2, OUT}, {f[3], kFeatBytes[3], S_F1 + 3, OUT},
                                        {t[0], kFeatBytes[0], S_T1, OUT}, {t[1], kFeatBytes[1], S_T1 + 1, OUT},
                                        {t[2], kFeatBytes[2], S_T1 + 2, OUT}, {t[3], kFeatBytes[3], S_T1 + 3, OUT}},
                   host ? ensure_introspect_plan<true, true> : ensure_introspect_plan<false, true>, [&](const Chunk& c) {
    int r = run_introspect_jvp(h, c.pl, c.f(0), c.f(1), c.st);
    float* o[4] = {c.f(2), c.f(3), c.f(4), c.f(5)};
    float* ot[4] = {c.f(6), c.f(7), c.f(8), c.f(9)};
    if (r == IAN_OK) r = store_features(h, c.pl, false, o, nullptr, 1, c.st);
    return r != IAN_OK ? r : store_features(h, c.pl, true, ot, nullptr, 1, c.st);
  });
}

// ---- the features' vector-Jacobian product (DESIGN section 5.6l) ---------------------------------------------------------
// dx = sum_i (d g_i / d x)^T c_i: run_encode_vjp's chain entered at the deepest supplied layer L instead of at the head.
// The forward stops after enc_conv{L}; feat_cotangent writes c_L times scale_L * lrelu'(a_L) into e_L -- exactly what the
// GEMM landing on a_L would write from a zero accumulator with c_L as res, so a zero c_L above gives the same bits as
// leaving it out -- and the shallower supplied c_l, as they are, into the staging planes ivc.  Each backward
// GEMM that lands on a layer with a supplied cotangent runs as its IV_BWD_* copy, whose epilogue adds ivc before the
// activation derivative: e_l = (acc + c_l) * scale_l * lrelu'(a_l) (res, res_after = 0, ACT_MASK, as the encoder JVP's
// tangent twins use it); a layer without one runs the encoder VJP's own descriptor.  enc_conv1's adjoint ends the chain.
// The first call on a plan allocates what ian_encode_vjp_* does (shared with it) and the staging planes; the host form
// stages x in the plan's image buffer, the cotangents in the ian_introspect*_host buffer and dx in its x_hat buffer.
template <bool kHost>
int ensure_introspect_vjp_plan(ian_handle* h, Plan* pl) {
  int rc;
  if ((rc = ensure_enc_vjp_plan(h, pl)) != IAN_OK) return rc;
  if (!pl->ivjp) {
    const Planes* a[3] = {&pl->a1, &pl->a2, &pl->a3};
    const int from[3] = {E_BWD_CONV2, E_BWD_CONV3, E_BWD_CONV4}, to[3] = {IV_BWD_CONV2, IV_BWD_CONV3, IV_BWD_CONV4};
    for (int l = 0; l < 3; ++l) {
      if ((rc = alloc_planes(h, pl, pl->ivc[l], a[l]->plane)) != IAN_OK) return rc;
      TapGemm& g = pl->g[to[l]];
      g = pl->g[from[l]];                                 // its split-K factor and slabs too: the two never run at once
      g.res = pl->ivc[l].p; g.res_plane = pl->ivc[l].plane; g.res_after = 0;
      char err[256] = {0};
      if (!(pl->maps[to[l]] = tc_build_maps(g, err, sizeof(err)))) return fail(h, IAN_ERR_CUDA, "layer %s: %s", kLayerNames[to[l]], err);
    }
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    pl->ivjp = true;
  }
  return ensure_introspect_plan<kHost, false>(h, pl);
}

int run_introspect_vjp(ian_handle* h, Plan* pl, const float* x, const float* const* c, float* dx, cudaStream_t st) {
  const int n = pl->n;
  int L = 4;                                              // the deepest supplied layer, 1-based
  while (L > 0 && !c[L - 1]) --L;
  if (L == 0) {
    CUDA_TRY(h, cudaMemsetAsync(dx, 0, (size_t)n * kImageBytes, st));
    return IAN_OK;
  }
  int rc = run_introspect(h, pl, x, st, L);
  if (rc != IAN_OK) return rc;
  Planes* e[4] = {&pl->e1, &pl->e2, &pl->e3, &pl->e4};
  FeatCotangents fc{};
  for (int l = 0; l < L; ++l) {
    fc.c[l] = c[l];
    const Planes& o = l == L - 1 ? *e[l] : pl->ivc[l];
    fc.out[l] = o.p;
    fc.plane[l] = o.plane;
  }
  fc.deep = L - 1;
  // e_L's lo plane as the GEMM landing on a_L leaves it: bf16 mode writes it only in a split-K finalize (tapgemm.h), and
  // enc_conv1's adjoint reads hi + lo of e1, in later encoder VJP calls too
  const int land[4] = {E_BWD_CONV2, E_BWD_CONV3, E_BWD_CONV4, E_BWD_FC1};
  fc.deep_lo = h->passes != 1 || (h->path == IAN_PATH_TC && pl->g[land[L - 1]].ksplit > 1);
  fc.mask = feat_planes(pl, L - 1).p;
  fc.scale = L == 1 ? nullptr : h->w[kEncoder.l[L - 2]].scale;   // bnorm{L}; enc_conv1 has a bias and no BatchNorm
  {
    ScopedTimer tm(h, T_FEAT_COTANGENT, st);
    LAUNCH_TRY(h, launch_feat_cotangent(fc, h->passes, n, st));
  }
  const int bwd[3][2] = {{E_BWD_CONV2, IV_BWD_CONV2}, {E_BWD_CONV3, IV_BWD_CONV3}, {E_BWD_CONV4, IV_BWD_CONV4}};
  for (int l = L - 2; l >= 0; --l)                        // e_{l+2} -> e_{l+1} (1-based), joined by c_{l+1}
    if ((rc = run_gemm(h, pl, bwd[l][c[l] ? 1 : 0], st)) != IAN_OK) return rc;
  ScopedTimer tm(h, T_CONV1_BWD, st);
  if (h->path == IAN_PATH_TC)
    LAUNCH_TRY(h, launch_conv1_bwd_tc(pl->conv1_bwd_maps, dx, n, st));
  else
    LAUNCH_TRY(h, launch_conv1_bwd(pl->e1.p, pl->e1.plane, h->conv1_bwd_wt, dx, n, st));
  return IAN_OK;
}

// No CUDA graphs, as for the other introspect entries.  All four cotangents NULL: dx = 0, nothing else runs.
int call_introspect_vjp(ian_handle* h, bool host, const float* x, int n, const float* const* c, float* dx, void* stream) {
  int rc = check_fit_args(h, n);
  if (rc != IAN_OK || n == 0) return rc;
  if (!x || !dx) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  const bool any = c[0] || c[1] || c[2] || c[3];
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {c[0], kFeatBytes[0], S_F1, IN},
                                        {c[1], kFeatBytes[1], S_F1 + 1, IN}, {c[2], kFeatBytes[2], S_F1 + 2, IN},
                                        {c[3], kFeatBytes[3], S_F1 + 3, IN}, {dx, kImageBytes, S_XHAT, OUT}},
                   !any ? nullptr : host ? ensure_introspect_vjp_plan<true> : ensure_introspect_vjp_plan<false>,
                   [&](const Chunk& ch) {
    const float* ct[4] = {ch.f(1), ch.f(2), ch.f(3), ch.f(4)};
    return run_introspect_vjp(h, ch.pl, ch.f(0), ct, ch.f(5), ch.st);
  });
}

// ---- the discriminator head l_discrim (DESIGN section 5.6n) ---------------------------------------------------------
// logits = [pool(a4) | f] W with f the MinibatchLayer's features of the pooled batch, p = sigmoid / softmax(logits), under
// deterministic=True.  The MinibatchLayer couples the samples of the call, so the entries run in phases: per chunk the trunk
// (run_introspect) and the pool into a whole-call buffer at the chunk's offset; over the whole call the MinibatchLayer and
// the dense layer (and, in the VJP, their adjoints); per chunk again the trunk's reverse chain from enc_conv4's cotangent.
// The minibatch is therefore the call's batch whatever IAN_CHUNK is.  No CUDA graphs, as for the introspect entries.
const char* const kDiscParams[4] = {"minibatch_discrim.theta", "minibatch_discrim.log_weight_scale", "minibatch_discrim.b",
                                    "discrimi.W"};
constexpr int kDiscIn = 1024 + kDiscKernels;
inline int disc_units(const ian_handle* h) { return h->model_kind == IAN_MODEL_FULL ? kDiscMaxUnits : 1; }

struct DiscBufs { float *pool, *in, *g, *dpool, *logits, *p, *dlogits, *c4; };
DiscBufs disc_bufs(ian_handle* h, int cap) {
  DiscBufs b;
  const long long N = cap;
  b.pool = h->disc_buf;
  b.in = b.pool + N * 1024;
  b.g = b.in + N * kDiscIn;
  b.dpool = b.g + N * kDiscIn;
  b.logits = b.dpool + N * 1024;
  b.p = b.logits + N * kDiscMaxUnits;
  b.dlogits = b.p + N * kDiscMaxUnits;
  b.c4 = b.dlogits + N * kDiscMaxUnits;
  return b;
}

int ensure_disc_bufs(ian_handle* h, int n, DiscBufs* out) {
  if (n > h->disc_cap) {
    CUDA_TRY(h, cudaDeviceSynchronize());
    CUDA_TRY(h, cudaFree(h->disc_buf));
    h->disc_buf = nullptr;
    h->disc_cap = 0;
    const long long N = n, chunk = std::min(n, h->max_chunk);
    CUDA_TRY(h, cudaMalloc((void**)&h->disc_buf, (size_t)(N * (2 * 1024 + 2 * kDiscIn + 3 * kDiscMaxUnits) + chunk * 16384) * sizeof(float)));
    h->disc_cap = n;
  }
  *out = disc_bufs(h, h->disc_cap);
  return IAN_OK;
}

int check_discriminate(ian_handle* h, int n) {
  const int rc = check_fit_args(h, n);
  if (rc != IAN_OK) return rc;
  if (h->disc_set != 15) return fail(h, IAN_ERR_STATE, "no discriminator head loaded (ian_set_discriminator_param)");
  return IAN_OK;
}

// phase 1: per chunk, the trunk to enc_conv4 and the pool of a4 into b.pool at the chunk's offset
int disc_pool_phase(ian_handle* h, bool host, const float* x, int n, const DiscBufs& b, void* stream) {
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}}, nullptr, [&](const Chunk& c) {
    const int r = run_introspect(h, c.pl, c.f(0), c.st);
    if (r != IAN_OK) return r;
    ScopedTimer tm(h, T_DISC_POOL, c.st);
    LAUNCH_TRY(h, launch_disc_pool(c.pl->a4.p, c.pl->a4.plane, h->passes, c.cn, b.pool + (size_t)c.off * 1024, c.st));
    return (int)IAN_OK;
  });
}

int call_discriminate(ian_handle* h, bool host, const float* x, int n, float* logits, float* p, void* stream) {
  int rc = check_discriminate(h, n);
  if (rc != IAN_OK || n == 0) return rc;
  if (!x || !logits) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  DeviceGuard dg(h->device);
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  const int U = disc_units(h);
  DiscBufs b;
  if ((rc = ensure_disc_bufs(h, n, &b)) != IAN_OK || (rc = ensure_train_ws(h, mb_workspace_bytes(n, kDiscKernels, kDiscDims))) != IAN_OK ||
      (rc = disc_pool_phase(h, host, x, n, b, stream)) != IAN_OK)
    return rc;
  float* lo = host ? b.logits : logits;
  float* po = !p ? nullptr : host ? b.p : p;
  {
    ScopedTimer tm(h, T_DISC_MB, st);
    LAUNCH_TRY(h, launch_minibatch_discrim(b.pool, n, 1024, h->disc_w[0], h->disc_w[1], h->disc_w[2], kDiscKernels, kDiscDims, b.in,
                                           h->train_ws, st));
  }
  {
    ScopedTimer tm(h, T_DISC_HEAD, st);
    LAUNCH_TRY(h, launch_disc_head(b.in, h->disc_w[3], U, n, lo, po, st));
  }
  if (!host) return IAN_OK;
  CUDA_TRY(h, cudaMemcpyAsync(logits, lo, (size_t)n * U * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (p) CUDA_TRY(h, cudaMemcpyAsync(p, po, (size_t)n * U * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaStreamSynchronize(st));
  return IAN_OK;
}

// phase 2 over the whole call, dlogits -> d[pool | f] -> d pool; phase 3 per chunk, c4 from d pool and run_introspect_vjp
// with c = {0, 0, 0, c4}.  The trunk's forward runs twice: 2 forwards and 1 backward.
int call_discriminate_vjp(ian_handle* h, bool host, const float* x, int n, const float* dlogits, float* dx, void* stream) {
  int rc = check_discriminate(h, n);
  if (rc != IAN_OK || n == 0) return rc;
  if (!x || !dlogits || !dx) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  DeviceGuard dg(h->device);
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  const int U = disc_units(h);
  DiscBufs b;
  if ((rc = ensure_disc_bufs(h, n, &b)) != IAN_OK ||
      (rc = ensure_train_ws(h, mb_bwd_workspace_bytes(n, 1024, kDiscKernels, kDiscDims))) != IAN_OK ||
      (rc = disc_pool_phase(h, host, x, n, b, stream)) != IAN_OK)
    return rc;
  const float* dl = dlogits;
  if (host) {
    CUDA_TRY(h, cudaMemcpyAsync(b.dlogits, dlogits, (size_t)n * U * sizeof(float), cudaMemcpyHostToDevice, st));
    dl = b.dlogits;
  }
  {
    ScopedTimer tm(h, T_DISC_HEAD_BWD, st);
    LAUNCH_TRY(h, launch_disc_head_bwd(dl, h->disc_w[3], U, n, b.g, st));
  }
  {
    ScopedTimer tm(h, T_DISC_MB_BWD, st);
    LAUNCH_TRY(h, launch_minibatch_discrim_bwd(b.pool, n, 1024, h->disc_w[0], h->disc_w[1], kDiscKernels, kDiscDims, b.g, b.dpool,
                                               nullptr, nullptr, nullptr, h->train_ws, st));
  }
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {dx, kImageBytes, S_XHAT, OUT}}, ensure_introspect_vjp_plan<false>,
                   [&](const Chunk& c) {
    {
      ScopedTimer tm(h, T_DISC_COTANGENT, c.st);
      LAUNCH_TRY(h, launch_disc_cotangent(b.dpool + (size_t)c.off * 1024, c.cn, b.c4, c.st));
    }
    const float* ct[4] = {nullptr, nullptr, nullptr, b.c4};
    return run_introspect_vjp(h, c.pl, c.f(0), ct, c.f(1), c.st);
  });
}

// ---- batch-statistics BatchNorm stacks (DESIGN section 5.6o) -----------------------------------------------------------
// The training-mode discriminator's trunk (bnorm2..4 on enc_conv2..4) and the IAN_simple decoder in training mode
// (bnorm_dec_fc2, bnorm_dc1..3 on l_dec_fc2, dec_conv1..3) normalise with the call's own statistics, so they couple the
// call's samples and run layer by layer over the whole call.  A BnStack holds what differs between the two as data; one set
// of helpers runs both.
// Forward, per layer: per chunk, the layer's twin (unit scale, no shift, no activation) writes its raw sums into a whole-call
// float32 buffer; over the call, per-image float64 sums added in image order give mean and inv_std (so no result depends
// on IAN_CHUNK); per chunk again bn_act normalises, activates and writes the next layer's input planes.
// Backward, from the top layer down: whole-call float64 Σdy, Σdy·x and the coefficients; then per chunk dx as split planes,
// the layer below's activation recomputed from its raw sums (the backward GEMM's mask) and the backward-data twin (unit
// scale, float32 output) into the next cotangent slot.  The bottom layer's dx and what follows it are the caller's.
struct BnStack {
  int id;                                   // its slots in ian_handle::bn_bufs and Plan::bn_twins
  int L, C[4], HW[4];                       // layers; each layer's channels and pixels
  int off[4], total;                        // each layer's columns in the concatenated stats and gamma | beta
  int fwd, fwd_of[4];                       // layer l's forward twin is fwd + l, a twin of fwd_of[l]
  int bwd, bwd_of[3];                       // the backward-data twin from layer L-1-k down: bwd + k, a twin of bwd_of[k]
  int (*vjp_plan)(ian_handle*, Plan*);      // the VJP planes the backward twins read and write
  float act_abs, act_lin;                   // the activation fmaf(act_abs, |y|, act_lin y), as the tap-GEMM epilogue forms it
  int t_stats, t_norm, t_bn_bwd, t_bn_dx;   // timer slots
  float* ian_handle::*gb;                   // gamma | beta, [2][total]
  Planes Plan::*act[4], Plan::*dx[4];       // layer l's activation planes (the next layer's input) and its dx planes
};
constexpr BnStack kDiscStack = {0, 3, {256, 512, 1024}, {256, 64, 16}, {0, 256, 768}, 1792,
                                DT_ENC_CONV2, {L_ENC_CONV2, L_ENC_CONV3, L_ENC_CONV4}, DT_BWD_CONV4, {E_BWD_CONV4, E_BWD_CONV3},
                                ensure_enc_vjp_plan, 0.4f, 0.6f,   // LeakyRectify(0.2)
                                T_DT_STATS, T_DT_NORM, T_DT_BN_BWD, T_DT_BN_DX, &ian_handle::enc_bn_gb,
                                {&Plan::a2, &Plan::a3, &Plan::a4}, {&Plan::e2, &Plan::e3, &Plan::e4}};
constexpr BnStack kDecStack = {1, 4, {16384, 512, 256, 128}, {1, 64, 256, 1024},
                               {kDecBnOff[0], kDecBnOff[1], kDecBnOff[2], kDecBnOff[3]}, kDecBnTotal,
                               DD_DEC_FC2, {L_DEC_FC2, L_DEC_CONV1, L_DEC_CONV2, L_DEC_CONV3},
                               DD_BWD_CONV3, {L_BWD_CONV3, L_BWD_CONV2, L_BWD_CONV1},
                               ensure_param_vjp_plan, 0.5f, 0.5f,   // rectify
                               T_DD_STATS, T_DD_NORM, T_DD_BN_BWD, T_DD_BN_DX, &ian_handle::dec_bn_gb,
                               {&Plan::h0, &Plan::h1, &Plan::h2, &Plan::h3}, {&Plan::d0, &Plan::d1, &Plan::d2, &Plan::d3}};
constexpr float kBnEps = 1e-4f;

long long bn_elems(const BnStack& S, int l) { return (long long)S.C[l] * S.HW[l]; }   // per image

// raw[l]: layer l's raw sums (n, HW, C).  dy: two cotangent slots, layer l's dy (n, HW, C) in dy[(L-1-l) % 2], each sized
// for its largest layer: layer l's dy is last read by its own dx step, so layer l-1's twin writes the other slot and only
// layer l-2's twin, after layer l is done, writes this one again.  part: the per-image partial sums [n][2][max C]; fsum,
// bsum: the forward's and the backward's [2][C] sums of layer l at 2 off[l]; coef: [4][max C]; stats: [2][total] float32,
// the means then the inv_std in the library's column order; sout: [2][total], the staging of a reordered copy of stats
struct BnBufs {
  float *raw[4], *dy[2], *stats, *sout;
  double *part, *fsum, *bsum, *coef;
};

float* bn_dy(const BnStack& S, const BnBufs& b, int l) { return b.dy[(S.L - 1 - l) % 2]; }

int ensure_bn_bufs(ian_handle* h, const BnStack& S, int n, BnBufs* b) {
  int maxc = 0;
  long long slot[2] = {0, 0}, per_img = 0;   // floats
  for (int l = 0; l < S.L; ++l) {
    maxc = std::max(maxc, S.C[l]);
    slot[(S.L - 1 - l) % 2] = std::max(slot[(S.L - 1 - l) % 2], bn_elems(S, l));
    per_img += bn_elems(S, l);
  }
  per_img += slot[0] + slot[1];
  auto& s = h->bn_bufs[S.id];
  if (n > s.cap) {
    CUDA_TRY(h, cudaDeviceSynchronize());
    CUDA_TRY(h, cudaFree(s.buf));
    s.buf = nullptr;
    s.cap = 0;
    const size_t bytes = (size_t)n * (per_img * sizeof(float) + 2 * maxc * sizeof(double)) +
                         (4 * S.total + 4 * maxc) * sizeof(double) + 4 * S.total * sizeof(float);
    CUDA_TRY(h, cudaMalloc((void**)&s.buf, bytes));
    s.cap = n;
  }
  const long long N = s.cap;
  b->part = (double*)s.buf;
  b->fsum = b->part + N * 2 * maxc;
  b->bsum = b->fsum + 2 * S.total;
  b->coef = b->bsum + 2 * S.total;
  b->stats = (float*)(b->coef + 4 * maxc);
  b->sout = b->stats + 2 * S.total;
  float* f = b->sout + 2 * S.total;
  for (int l = 0; l < S.L; ++l) { b->raw[l] = f; f += N * bn_elems(S, l); }
  b->dy[0] = f;
  b->dy[1] = f + N * slot[0];
  return IAN_OK;
}

// the twins share the originals' B tiles, taps and split-K slabs (the two never run at once); only the epilogue differs
int build_twin(ian_handle* h, Plan* pl, int to, int from) {
  TapGemm& g = pl->g[to];
  g = pl->g[from];
  g.scale = nullptr; g.shift = nullptr; g.out = nullptr; g.out_plane = 0; g.out_f32 = nullptr; g.scale_pix_stride = 0;
  if (g.act != ACT_MASK) g.act = ACT_NONE;
  char err[256] = {0};
  if (!(pl->maps[to] = tc_build_maps(g, err, sizeof(err)))) return fail(h, IAN_ERR_CUDA, "layer %s: %s", kLayerNames[to], err);
  return IAN_OK;
}

// the stack's forward twins on the plan; with vjp also its backward-data twins, on the VJP's planes
int ensure_bn_twins(ian_handle* h, Plan* pl, const BnStack& S, bool vjp) {
  bool* built = pl->bn_twins[S.id];
  int rc;
  if (!built[0]) {
    for (int l = 0; l < S.L; ++l)
      if ((rc = build_twin(h, pl, S.fwd + l, S.fwd_of[l])) != IAN_OK) return rc;
    built[0] = true;
  }
  if (vjp && !built[1]) {
    if ((rc = S.vjp_plan(h, pl)) != IAN_OK) return rc;
    for (int k = 0; k < S.L - 1; ++k)
      if ((rc = build_twin(h, pl, S.bwd + k, S.bwd_of[k])) != IAN_OK) return rc;
    built[1] = true;
  }
  return IAN_OK;
}

// ensure_bn_twins as run_entry's prepare
template <const BnStack& S, bool kVjp>
int ensure_bn_plan(ian_handle* h, Plan* pl) { return ensure_bn_twins(h, pl, S, kVjp); }

int run_gemm_into(ian_handle* h, Plan* pl, int l, float* out, cudaStream_t st) {
  pl->g[l].out_f32 = out;
  return run_gemm(h, pl, l, st);
}

// layer l's batch-normalised, activated output of the chunk at `off` -> its activation planes
int bn_act(ian_handle* h, const BnStack& S, const BnBufs& b, int l, Plan* pl, int off, int cn, cudaStream_t st) {
  ScopedTimer tm(h, S.t_norm, st);
  const float* gb = h->*S.gb + S.off[l];
  const Planes& a = pl->*S.act[l];
  LAUNCH_TRY(h, launch_nhwc_bn_act(b.raw[l] + off * bn_elems(S, l), cn * bn_elems(S, l), S.C[l], b.stats + S.off[l],
                                   b.stats + S.total + S.off[l], gb, gb + S.total, S.act_abs, S.act_lin, h->passes, a.p,
                                   a.plane, st));
  return IAN_OK;
}

// forward: layer l's sums into b.fsum and its statistics into b.stats; backward: Σdy, Σdy·x into b.bsum, then the coefficients
int bn_sums(ian_handle* h, const BnStack& S, const BnBufs& b, int l, int n, bool bwd, cudaStream_t st) {
  const double count = (double)n * S.HW[l];
  const int C = S.C[l], o = S.off[l];
  ScopedTimer tm(h, bwd ? S.t_bn_bwd : S.t_stats, st);
  if (!bwd) {
    LAUNCH_TRY(h, launch_nhwc_bn_sums(b.raw[l], b.raw[l], n, S.HW[l], C, count, kBnEps, b.part, b.fsum + 2 * o, b.stats + o,
                                      b.stats + S.total + o, st));
    return IAN_OK;
  }
  LAUNCH_TRY(h, launch_nhwc_bn_sums(bn_dy(S, b, l), b.raw[l], n, S.HW[l], C, 0.0, kBnEps, b.part, b.bsum + 2 * o, nullptr, nullptr,
                                    st));
  LAUNCH_TRY(h, launch_nhwc_bn_coef(b.fsum + 2 * o, b.bsum + 2 * o, count, kBnEps, h->*S.gb + o, C, b.coef, st));
  return IAN_OK;
}

// dL/d(raw sum) of layer l for the chunk at `off`, from its dy and the coefficients -> its dx planes
int bn_dx(ian_handle* h, const BnStack& S, const BnBufs& b, int l, Plan* pl, int off, int cn, cudaStream_t st) {
  ScopedTimer tm(h, S.t_bn_dx, st);
  const Planes& d = pl->*S.dx[l];
  const long long e = bn_elems(S, l);
  LAUNCH_TRY(h, launch_nhwc_bn_dx(b.raw[l] + off * e, bn_dy(S, b, l) + off * e, cn * e, S.C[l], b.coef, h->passes, d.p, d.plane,
                                  st));
  return IAN_OK;
}

// the forward to every layer's raw sums and statistics; first(c) writes the chunk's input planes of layer 0's twin.  The
// top layer's activation is the caller's, per chunk.
template <const BnStack& S, bool kVjp, typename First>
int bn_forward(ian_handle* h, bool host, const Arg& in, int n, const BnBufs& b, void* stream, First&& first) {
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  int rc = run_entry(h, host, stream, n, {in}, ensure_bn_plan<S, kVjp>, [&](const Chunk& c) {
    const int r = first(c);
    return r != IAN_OK ? r : run_gemm_into(h, c.pl, S.fwd, b.raw[0] + c.off * bn_elems(S, 0), c.st);
  });
  if (rc != IAN_OK || (rc = bn_sums(h, S, b, 0, n, false, st)) != IAN_OK) return rc;
  for (int l = 1; l < S.L; ++l) {
    rc = for_chunks(h, n, [&](Plan* pl, int off, int cn) {
      int r = ensure_bn_twins(h, pl, S, kVjp);
      if (r == IAN_OK) r = bn_act(h, S, b, l - 1, pl, off, cn, st);
      return r != IAN_OK ? r : run_gemm_into(h, pl, S.fwd + l, b.raw[l] + off * bn_elems(S, l), st);
    });
    if (rc != IAN_OK || (rc = bn_sums(h, S, b, l, n, false, st)) != IAN_OK) return rc;
  }
  return IAN_OK;
}

// the backward from the top layer's dy, in its slot, to the bottom layer's coefficients.  hook(pl, l, off, cn) runs per
// chunk once layer l's dx planes and layer l-1's activation planes are written, before the backward-data twin.
template <typename Hook>
int bn_backward(ian_handle* h, const BnStack& S, const BnBufs& b, int n, cudaStream_t st, Hook&& hook) {
  int rc;
  for (int l = S.L - 1; l >= 1; --l) {
    if ((rc = bn_sums(h, S, b, l, n, true, st)) != IAN_OK) return rc;
    rc = for_chunks(h, n, [&](Plan* pl, int off, int cn) {
      int r = ensure_bn_twins(h, pl, S, true);
      if (r == IAN_OK) r = bn_dx(h, S, b, l, pl, off, cn, st);
      if (r == IAN_OK) r = bn_act(h, S, b, l - 1, pl, off, cn, st);
      if (r == IAN_OK) r = hook(pl, l, off, cn);
      return r != IAN_OK ? r : run_gemm_into(h, pl, S.bwd + (S.L - 1 - l), bn_dy(S, b, l - 1) + off * bn_elems(S, l - 1), st);
    });
    if (rc != IAN_OK) return rc;
  }
  return bn_sums(h, S, b, 0, n, true, st);
}

// ---- the discriminator in training mode (DESIGN section 5.6o) ----------------------------------------------------------
// l_discrim under deterministic=False: enc_conv1 as ever, then kDiscStack, a4's pool and the head as in inference.  The VJP
// keeps the forward's raw buffers: the head's and the MinibatchLayer's adjoints, then the pool's adjoint times lrelu'(y4) as
// bnorm4's dy, the stack's backward, and per chunk bnorm2's dx, enc_conv2's backward (its scale is 1 already) and
// enc_conv1's adjoint.

// the whole forward to the pooled features d.pool
template <bool kVjp>
int disc_train_trunk(ian_handle* h, bool host, const float* x, int n, const DiscBufs& d, const BnBufs& b, void* stream) {
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  int rc = bn_forward<kDiscStack, kVjp>(h, host, {x, kImageBytes, S_X, IN}, n, b, stream,
                                        [&](const Chunk& c) { return run_introspect(h, c.pl, c.f(0), c.st, 1); });
  if (rc != IAN_OK) return rc;
  return for_chunks(h, n, [&](Plan* pl, int off, int cn) {
    const int r = bn_act(h, kDiscStack, b, 2, pl, off, cn, st);
    if (r != IAN_OK) return r;
    ScopedTimer tm(h, T_DISC_POOL, st);
    LAUNCH_TRY(h, launch_disc_pool(pl->a4.p, pl->a4.plane, h->passes, cn, d.pool + (size_t)off * 1024, st));
    return (int)IAN_OK;
  });
}

int call_discriminate_train(ian_handle* h, bool host, const float* x, int n, float* logits, float* p, float* stats, void* stream) {
  int rc = check_discriminate(h, n);
  if (rc != IAN_OK || n == 0) return rc;
  if (!x || !logits) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  DeviceGuard dg(h->device);
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  const int U = disc_units(h);
  DiscBufs d;
  BnBufs b;
  if ((rc = ensure_disc_bufs(h, n, &d)) != IAN_OK || (rc = ensure_bn_bufs(h, kDiscStack, n, &b)) != IAN_OK ||
      (rc = ensure_train_ws(h, mb_workspace_bytes(n, kDiscKernels, kDiscDims))) != IAN_OK ||
      (rc = disc_train_trunk<false>(h, host, x, n, d, b, stream)) != IAN_OK)
    return rc;
  float* lo = host ? d.logits : logits;
  float* po = !p ? nullptr : host ? d.p : p;
  {
    ScopedTimer tm(h, T_DISC_MB, st);
    LAUNCH_TRY(h, launch_minibatch_discrim(d.pool, n, 1024, h->disc_w[0], h->disc_w[1], h->disc_w[2], kDiscKernels, kDiscDims, d.in,
                                           h->train_ws, st));
  }
  {
    ScopedTimer tm(h, T_DISC_HEAD, st);
    LAUNCH_TRY(h, launch_disc_head(d.in, h->disc_w[3], U, n, lo, po, st));
  }
  const cudaMemcpyKind k = host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  if (stats) CUDA_TRY(h, cudaMemcpyAsync(stats, b.stats, 2 * kDiscStack.total * sizeof(float), k, st));
  if (!host) return IAN_OK;
  CUDA_TRY(h, cudaMemcpyAsync(logits, lo, (size_t)n * U * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (p) CUDA_TRY(h, cudaMemcpyAsync(p, po, (size_t)n * U * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaStreamSynchronize(st));
  return IAN_OK;
}

// 1 forward + 1 backward: the forward's raw buffers stay for the backward, whose masks are recomputed per chunk from them
int call_discriminate_train_vjp(ian_handle* h, bool host, const float* x, int n, const float* dlogits, float* dx, void* stream) {
  int rc = check_discriminate(h, n);
  if (rc != IAN_OK || n == 0) return rc;
  if (!x || !dlogits || !dx) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  DeviceGuard dg(h->device);
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  const int U = disc_units(h);
  const BnStack& S = kDiscStack;
  DiscBufs d;
  BnBufs b;
  if ((rc = ensure_disc_bufs(h, n, &d)) != IAN_OK || (rc = ensure_bn_bufs(h, S, n, &b)) != IAN_OK ||
      (rc = ensure_train_ws(h, mb_bwd_workspace_bytes(n, 1024, kDiscKernels, kDiscDims))) != IAN_OK ||
      (rc = disc_train_trunk<true>(h, host, x, n, d, b, stream)) != IAN_OK)
    return rc;
  const float* dl = dlogits;
  if (host) {
    CUDA_TRY(h, cudaMemcpyAsync(d.dlogits, dlogits, (size_t)n * U * sizeof(float), cudaMemcpyHostToDevice, st));
    dl = d.dlogits;
  }
  {
    ScopedTimer tm(h, T_DISC_HEAD_BWD, st);
    LAUNCH_TRY(h, launch_disc_head_bwd(dl, h->disc_w[3], U, n, d.g, st));
  }
  {
    ScopedTimer tm(h, T_DISC_MB_BWD, st);
    LAUNCH_TRY(h, launch_minibatch_discrim_bwd(d.pool, n, 1024, h->disc_w[0], h->disc_w[1], kDiscKernels, kDiscDims, d.g, d.dpool,
                                               nullptr, nullptr, nullptr, h->train_ws, st));
  }
  {
    ScopedTimer tm(h, T_DT_COTANGENT, st);
    const float* gb = h->enc_bn_gb + S.off[2];
    LAUNCH_TRY(h, launch_disc_train_cotangent(d.dpool, b.raw[2], n, b.stats + S.off[2], b.stats + S.total + S.off[2], gb,
                                              gb + S.total, bn_dy(S, b, 2), st));
  }
  if ((rc = bn_backward(h, S, b, n, st, [](Plan*, int, int, int) { return (int)IAN_OK; })) != IAN_OK) return rc;
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {dx, kImageBytes, S_XHAT, OUT}}, ensure_bn_plan<kDiscStack, true>,
                   [&](const Chunk& c) {
    int r = bn_dx(h, S, b, 0, c.pl, c.off, c.cn, c.st);
    if (r == IAN_OK) r = run_introspect(h, c.pl, c.f(0), c.st, 1);     // a1: the mask of enc_conv2's backward
    if (r == IAN_OK) r = run_gemm(h, c.pl, E_BWD_CONV2, c.st);
    if (r != IAN_OK) return r;
    ScopedTimer tm(h, T_CONV1_BWD, c.st);
    if (h->path == IAN_PATH_TC)
      LAUNCH_TRY(h, launch_conv1_bwd_tc(c.pl->conv1_bwd_maps, c.f(1), c.cn, c.st));
    else
      LAUNCH_TRY(h, launch_conv1_bwd(c.pl->e1.p, c.pl->e1.plane, h->conv1_bwd_wt, c.f(1), c.cn, c.st));
    return (int)IAN_OK;
  });
}

// ---- the IAN_simple decoder in training mode (DESIGN section 5.6p) ----------------------------------------------------
// get_output(l_out, {l_Z: z}) under deterministic=False: kDecStack on the latent planes, then dec_out as ever on h3.  The VJP
// runs that forward, then per chunk the parameter VJP's dense seed (the seed image and dL/dh3 before the mask), dec_out's
// weight gradient and bnorm_dc3's dy; the stack's backward with each layer's weight gradient (wgrad on its dx planes and its
// training-mode input, chunks added in order) as the hook; d beta and d gamma from the kept sums; and per chunk
// bnorm_dec_fc2's dx, l_dec_fc2's weight gradient and L_BWD_FC2 itself (unit scale already) for dz.

// the forward to every layer's raw sums and statistics (h3's planes are left to the caller, per chunk)
template <bool kVjp>
int dec_train_forward(ian_handle* h, bool host, const float* z, int n, const BnBufs& b, void* stream) {
  return bn_forward<kDecStack, kVjp>(h, host, {z, kLatentBytes, S_Z, IN}, n, b, stream, [&](const Chunk& c) {
    LAUNCH_TRY(h, launch_z_to_planes(c.f(0), c.pl->zp.p, c.pl->zp.plane, c.cn, c.st));
    return (int)IAN_OK;
  });
}

int check_decode_train(ian_handle* h, int n) {
  if (!h) return IAN_ERR_INVALID;
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "ian_finalize() has not been called");
  if (h->model_kind != IAN_MODEL_SIMPLE)
    return fail(h, IAN_ERR_UNSUPPORTED, "the training-mode decoder is implemented for IAN_simple only");
  if (n < 0) return fail(h, IAN_ERR_INVALID, "batch size must not be negative (got %d)", n);
  return IAN_OK;
}

int call_decode_train(ian_handle* h, bool host, const float* z, int n, float* x_hat, float* stats, void* stream) {
  int rc = check_decode_train(h, n);
  if (rc != IAN_OK || n == 0) return rc;
  if (!z || !x_hat) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  DeviceGuard dg(h->device);
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  BnBufs b;
  if ((rc = ensure_bn_bufs(h, kDecStack, n, &b)) != IAN_OK || (rc = dec_train_forward<false>(h, host, z, n, b, stream)) != IAN_OK)
    return rc;
  if (stats) {
    LAUNCH_TRY(h, launch_dec_stats_out(b.stats, kDecBnTotal, 16384, host ? b.sout : stats, st));
    if (host) CUDA_TRY(h, cudaMemcpyAsync(stats, b.sout, 2 * kDecBnTotal * sizeof(float), cudaMemcpyDeviceToHost, st));
  }
  return run_entry(h, host, stream, n, {{x_hat, kImageBytes, S_XHAT, OUT}}, ensure_bn_plan<kDecStack, false>, [&](const Chunk& c) {
    const int r = bn_act(h, kDecStack, b, 3, c.pl, c.off, c.cn, c.st);
    return r != IAN_OK ? r : run_dec_out(h, c.pl, c.f(0), c.st);
  });
}

// 1 forward + 1 backward.  The host form computes the requested gradients into the handle's device buffers and copies them
// out at the end.
int call_decode_train_vjp(ian_handle* h, bool host, const float* z, const float* dx_hat, int n, float* dz, float* const* grads,
                          void* stream) {
  float* req[PV_COUNT];
  int rc = check_param_vjp(h, z, dx_hat, n, grads, req);
  if (rc != IAN_OK || n == 0) return rc;
  DeviceGuard dg(h->device);
  const cudaStream_t st = !host && stream ? (cudaStream_t)stream : h->stream;
  float* out[PV_COUNT];
  for (int k = 0; k < PV_COUNT; ++k) {
    out[k] = req[k];
    if (!host || !req[k]) continue;
    if (!h->pv_dev[k]) CUDA_TRY(h, cudaMalloc((void**)&h->pv_dev[k], (size_t)kPvSize[k] * 4));
    out[k] = h->pv_dev[k];
  }
  const BnStack& S = kDecStack;
  BnBufs b;
  if ((rc = ensure_bn_bufs(h, S, n, &b)) != IAN_OK || (rc = dec_train_forward<true>(h, host, z, n, b, stream)) != IAN_OK)
    return rc;
  // h3, x_hat and the seed per chunk: dec_out's weight gradient, and bnorm_dc3's dy from dL/dh3 and the training-mode mask
  rc = run_entry(h, host, stream, n, {{dx_hat, kImageBytes, S_TARGET, IN}}, ensure_bn_plan<kDecStack, true>, [&](const Chunk& c) {
    Plan* pl = c.pl;
    int r = bn_act(h, S, b, 3, pl, c.off, c.cn, c.st);
    if (r == IAN_OK) r = run_dec_out(h, pl, pl->xhat, c.st);
    if (r != IAN_OK) return r;
    {
      ScopedTimer tm(h, T_BRUSH_SEED, c.st);
      LAUNCH_TRY(h, launch_brush_param_seed_bwd(pl->xhat, c.f(0), h->decout_wt, h->w[L_DEC_CONV3].scale, pl->h3.p, pl->d3.p,
                                                pl->d3.plane, pl->pseed, pl->dh3.p, c.cn, c.st));
    }
    if (out[PV_OUT]) {
      ScopedTimer tm(h, T_WGRAD_DEC_OUT, c.st);
      LAUNCH_TRY(h, launch_decout_wgrad(pl->pseed, pl->h3.p, pl->h3.plane, c.cn, pl->ppart, out[PV_OUT], c.off > 0, c.st));
    }
    ScopedTimer tm(h, T_DD_COTANGENT, c.st);
    const float* gb = h->dec_bn_gb + S.off[3];
    const long long e = bn_elems(S, 3);
    LAUNCH_TRY(h, launch_dec_train_dy(pl->dh3.p, pl->dh3.plane, b.raw[3] + c.off * e, c.cn * e, S.C[3], b.stats + S.off[3],
                                      b.stats + S.total + S.off[3], gb, gb + S.total, bn_dy(S, b, 3) + c.off * e, c.st));
    return (int)IAN_OK;
  });
  if (rc != IAN_OK) return rc;
  // layer l's weight gradient from its dx planes and its input planes
  auto wgrad = [&](Plan* pl, int l, int off, int) {
    if (!out[PV_FC2 + l]) return (int)IAN_OK;
    {
      ScopedTimer tm(h, T_WGRAD_FC2 + l, st);
      if (h->path == IAN_PATH_TC) LAUNCH_TRY(h, launch_wgrad_tc(pl->wg[l], pl->wmaps[l], st));
      else LAUNCH_TRY(h, launch_wgrad_simt(pl->wg[l], st));
    }
    LAUNCH_TRY(h, launch_wgrad_finalize(pl->wg[l], l == 0 ? WG_FC2 : WG_DECONV, out[PV_FC2 + l], off > 0, st));
    return (int)IAN_OK;
  };
  if ((rc = bn_backward(h, S, b, n, st, wgrad)) != IAN_OK) return rc;
  for (int l = 0; l < S.L; ++l) {
    float *db = out[PV_BN0_B + 2 * l], *dg = out[PV_BN0_G + 2 * l];
    if (!db && !dg) continue;
    ScopedTimer tm(h, T_DD_BN_GRADS, st);
    LAUNCH_TRY(h, launch_dec_bn_grads(b.fsum + 2 * S.off[l], b.bsum + 2 * S.off[l], (double)n * S.HW[l], kBnEps, S.C[l], l == 0 ? 1 : 0,
                                      db, dg, st));
  }
  rc = run_entry(h, host, stream, n, {{z, kLatentBytes, S_Z, IN}}, ensure_bn_plan<kDecStack, true>, [&](const Chunk& c) {
    LAUNCH_TRY(h, launch_z_to_planes(c.f(0), c.pl->zp.p, c.pl->zp.plane, c.cn, c.st));
    int r = bn_dx(h, S, b, 0, c.pl, c.off, c.cn, c.st);
    if (r == IAN_OK) r = wgrad(c.pl, 0, c.off, c.cn);
    if (r == IAN_OK) r = run_gemm(h, c.pl, L_BWD_FC2, c.st);
    return r != IAN_OK ? r : copy_dz(c, dz);
  });
  if (rc != IAN_OK || !host) return rc;
  for (int k = 0; k < PV_COUNT; ++k)
    if (req[k]) CUDA_TRY(h, cudaMemcpyAsync(req[k], out[k], (size_t)kPvSize[k] * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaStreamSynchronize(st));
  return IAN_OK;
}

// E(z) = a |x_hat - x|^2 + sum_l c_l |g_l(x_hat) - g_l(x)|^2 with c_l = 3072 b / M_l (b * 12288 * l_f, l_f the per-sample
// feature loss of train_IAN.py:244).  J_l = (d g_l / d x)(x_hat) J comes from the truncated encoder JVP on the batch-100
// plan, with the decoder JVP's 100 rows x_hat as primal and J's columns as tangents.  The stored features g(x) and
// g(x_hat) come from encoder forwards on the caller's plan.  The first call on a handle also allocates the Gram's 11.2 MB of
// partials and the batch-100 plan's encoder tangent planes; the first call on a plan its 1.97 MB per image of features.
int ensure_feat_plan(ian_handle* h, Plan* pl) {
  int rc = ensure_gn_plan(h, pl);
  if (rc != IAN_OK) return rc;
  Plan* jp = nullptr;
  if ((rc = get_plan(h, 100, &jp)) != IAN_OK || (rc = ensure_enc_jvp_plan(h, jp)) != IAN_OK) return rc;
  if (!h->feat_part) CUDA_TRY(h, cudaMalloc((void**)&h->feat_part, feat_part_doubles() * sizeof(double)));
  if (pl->feat) return IAN_OK;
  const long long N = pl->n;
  if ((rc = alloc_buf(h, pl, pl->ftg, N * kFeatTotal)) != IAN_OK || (rc = alloc_buf(h, pl, pl->fcur, N * kFeatTotal)) != IAN_OK)
    return rc;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  pl->feat = true;
  return IAN_OK;
}

// the trial planes (the plan's a1..a4) against the plan's target features, current features kept in fcur
FeatLayers plan_feat_layers(Plan* pl) {
  FeatLayers f{};
  for (int l = 0; l < 4; ++l) {
    f.tan[l] = feat_planes(pl, l).p;
    f.plane[l] = feat_planes(pl, l).plane;
    f.cur[l] = pl->fcur + pl->n * kFeatOff[l];
    f.tgt[l] = pl->ftg + pl->n * kFeatOff[l];
  }
  return f;
}

int check_feat_weights(ian_handle* h, double a, double b) {
  if (!(a >= 0.0) || !std::isfinite(a)) return fail(h, IAN_ERR_INVALID, "pixel_weight must be finite and >= 0 (got %g)", a);
  if (!(b >= 0.0) || !std::isfinite(b)) return fail(h, IAN_ERR_INVALID, "feature_weight must be finite and >= 0 (got %g)", b);
  if (a == 0.0 && b == 0.0) return fail(h, IAN_ERR_INVALID, "pixel_weight and feature_weight are both 0");
  return IAN_OK;
}

// ---- one driver for every latent fit (DESIGN section 5.6i) ---------------------------------------------------------------
// run_lm runs every objective: a start decode and an init accept, then per step the normal equations, the damped solve,
// a trial decode and the accept rule.  Each entry builds a Fit and runs one of two bodies, call_normal_eqs or call_fit.

// The objective of one fit entry, built once per call from its arguments; the kind picks the Gram and the accept kernel.
//   PLAIN     E(z) = |x_hat - x|^2                                       gn_gram, gn_accept
//   MAP       E(u) = sum_p w_p r_p^2 + beta |u|^2                          map_gram, map_accept
//   ROBUST    E(u) = sum_p w_p rho(r_p^2) + beta |u|^2, rho at scale dl     robust_gram, robust_accept
//   FEATURES  E(z) = a |x_hat - x|^2 + sum_l c_l |g_l(x_hat) - g_l(x)|^2     gn_gram (a != 0) + feat_gram, feat_accept
// w and dl are the chunk's (fit_at).
struct Fit {
  enum Kind { PLAIN, MAP, ROBUST, FEATURES } kind;
  bool flow = false;          // x_hat = decode(F(u)): MAP and ROBUST on the flow graphs
  double beta = 0.0;
  int loss = 0;               // ROBUST: IAN_ROBUST_HUBER or IAN_ROBUST_CAUCHY
  FeatWeights fw{};
  const float* w = nullptr;   // MAP, ROBUST: pixel weights, nullable
  double* dl = nullptr;       // ROBUST: the per-sample scale, the caller's or (automatic) robust_scale's from the start
  bool automatic = false;
  bool feats() const { return kind == FEATURES && fw.c[0] != 0.0; }
};
int (*const kFitPlan[4])(ian_handle*, Plan*) = {ensure_gn_plan, ensure_map_plan, ensure_robust_plan, ensure_feat_plan};

// c_l = 3072 b / M_l (b * 12288 * l_f, l_f the per-sample feature loss of train_IAN.py:244).  a = 1, b = 0 is the plain fit.
Fit feature_fit(double a, double b) {
  if (a == 1.0 && b == 0.0) return Fit{Fit::PLAIN};
  Fit f{Fit::FEATURES};
  f.fw.a = a;
  for (int l = 0; l < 4; ++l) f.fw.c[l] = 3072.0 * b / (double)feat_m(l);
  return f;
}

// fit with the chunk's pixel weights (Arg iw) and robust scale: the caller's (Arg is), or automatic into scale_out (Arg io;
// the plan's when left out).  In the host form both stage in the plan's scale buffer.
Fit fit_at(const Fit& fit, const Chunk& c, int iw, int is, int io) {
  Fit f = fit;
  double* s = (double*)c.p[is];
  double* o = (double*)c.p[io];
  f.w = c.f(iw);
  f.dl = s ? s : o ? o : c.pl->rdl;
  f.automatic = !s;
  return f;
}

// x_hat = decode(u) of the plan's n samples; with f.flow decode(F(u)), made_iaf_kernel writing the latent planes as
// `sample` does, so x_hat has ian_flow_*'s bits with x_out at that batch size
int fit_decode(ian_handle* h, Plan* pl, const Fit& f, const float* u, float* xo, cudaStream_t st) {
  if (!f.flow) return run_decode(h, pl, u, xo, st);
  LAUNCH_TRY(h, launch_made_iaf(u, h->made_w, h->made_b, nullptr, pl->zp.p, pl->zp.plane, pl->n, st));
  return run_decode_from_planes(h, pl, xo, st);
}

// the feature fit's target features, of x, into the plan's ftg
int feat_targets(ian_handle* h, Plan* pl, const float* x, cudaStream_t st) {
  const int rc = run_introspect(h, pl, x, st);
  return rc != IAN_OK ? rc : store_features(h, pl, false, nullptr, pl->ftg, 0, st);
}

// the robust fit's automatic scale, from x_hat and x of n samples
int robust_scale(ian_handle* h, const Fit& f, const float* xh, const float* x, int n, cudaStream_t st) {
  if (f.kind != Fit::ROBUST || !f.automatic) return IAN_OK;
  ScopedTimer tm(h, T_ROBUST_SCALE, st);
  LAUNCH_TRY(h, launch_robust_scale(xh, x, f.w, f.loss, f.dl, n, st));
  return IAN_OK;
}

// A (n,100,100), g (n,100) and e (n) of the plan's n samples at u, with x_hat already in xh and, for the feature fit with
// b != 0, the features of x and x_hat in the plan's ftg and fcur.  The robust Gram does not write e: its corner is not E.
int fit_normal_eqs(ian_handle* h, Plan* pl, const Fit& f, const float* u, const float* x, const float* xh, double* A,
                   double* g, double* e, cudaStream_t st) {
  Plan* jp = nullptr;
  int rc = get_plan(h, 100, &jp);
  if (rc != IAN_OK) return rc;
  const bool feats = f.feats();
  for (int k = 0; k < pl->n; ++k) {
    const float *uk = u + (size_t)k * 100, *xk = x + (size_t)k * 12288, *xhk = xh + (size_t)k * 12288;
    const float* wk = f.w ? f.w + (size_t)k * 12288 : nullptr;
    double *Ak = A + (size_t)k * 10000, *gk = g + (size_t)k * 100, *ek = e + k;
    const float *zr = h->gn_zrep, *tan = h->gn_eye;
    LAUNCH_TRY(h, launch_gn_replicate(uk, h->gn_zrep, st));
    if (f.flow) {
      zr = h->map_flow;
      tan = h->map_flow + 10000;
      LAUNCH_TRY(h, launch_made_iaf(h->gn_zrep, h->made_w, h->made_b, h->map_flow, nullptr, 0, 100, st));
      LAUNCH_TRY(h, launch_made_iaf_tangent(h->gn_zrep, h->gn_eye, h->made_w, h->made_b, h->map_flow + 10000, 100, st));
    }
    if ((rc = run_decode_jvp(h, jp, zr, tan, jp->xhat, h->gn_J, st)) != IAN_OK) return rc;
    if (f.kind == Fit::MAP) {
      ScopedTimer tm(h, T_MAP_GRAM, st);
      LAUNCH_TRY(h, launch_map_gram(h->gn_J, xhk, xk, wk, f.beta, uk, h->gn_part, Ak, gk, ek, st));
    } else if (f.kind == Fit::ROBUST) {
      ScopedTimer tm(h, T_ROBUST_GRAM, st);
      LAUNCH_TRY(h, launch_robust_gram(h->gn_J, xhk, xk, wk, f.loss, f.dl + k, f.beta, uk, h->gn_part, Ak, gk, st));
    } else if (f.kind == Fit::PLAIN || f.fw.a != 0.0) {
      ScopedTimer tm(h, T_GN_GRAM, st);
      LAUNCH_TRY(h, launch_gn_gram(h->gn_J, xhk, xk, h->gn_part, Ak, gk, ek, st));
    }
    if (f.kind != Fit::FEATURES) continue;
    FeatLayers t{};
    if (feats) {
      if ((rc = run_introspect_jvp(h, jp, jp->xhat, h->gn_J, st)) != IAN_OK) return rc;
      for (int l = 0; l < 4; ++l) {
        t.tan[l] = jp->jea[l].p;
        t.plane[l] = jp->jea[l].plane;
        t.cur[l] = pl->fcur + pl->n * kFeatOff[l] + k * feat_m(l);
        t.tgt[l] = pl->ftg + pl->n * kFeatOff[l] + k * feat_m(l);
      }
    }
    ScopedTimer tm(h, T_FEAT_GRAM, st);
    LAUNCH_TRY(h, launch_feat_gram(t, f.fw, feats, h->passes, f.fw.a != 0.0, h->feat_part, Ak, gk, ek, st));
  }
  return IAN_OK;
}

// the kind's accept kernel on the plan's n samples: E of the trial (x_hat_trial in fxt, u_trial in fzt), or with init of
// the start (x_hat in fxh), and the Levenberg-Marquardt decision on e, the plan's lambda and loss column col
int fit_accept(ian_handle* h, Plan* pl, const Fit& f, int init, const float* x, double* e, float* u, float* loss,
               long long ldl, int col, cudaStream_t st) {
  const float* xht = init ? pl->fxh : pl->fxt;
  const float* ut = init ? nullptr : pl->fzt;
  const int* ok = init ? nullptr : pl->fok;
  const int n = pl->n;
  switch (f.kind) {
    case Fit::PLAIN:
      LAUNCH_TRY(h, launch_gn_accept(init, xht, x, pl->fxh, e, pl->flam, u, ut, ok, loss, ldl, col, n, st));
      break;
    case Fit::MAP:
      LAUNCH_TRY(h, launch_map_accept(init, xht, x, f.w, f.beta, pl->fxh, e, pl->flam, u, ut, ok, loss, ldl, col, n, st));
      break;
    case Fit::ROBUST:
      LAUNCH_TRY(h, launch_robust_accept(init, xht, x, f.w, f.beta, f.loss, f.dl, pl->fxh, e, pl->flam, u, ut, ok, loss, ldl,
                                         col, n, st));
      break;
    case Fit::FEATURES: {
      ScopedTimer tm(h, T_FEAT_ACCEPT, st);
      LAUNCH_TRY(h, launch_feat_accept(init, xht, x, plan_feat_layers(pl), f.fw, f.feats(), h->passes, pl->fxh, e, pl->flam,
                                       u, ut, ok, loss, ldl, col, n, st));
    }
  }
  return IAN_OK;
}

// iters Levenberg-Marquardt steps in place on u (pl->n samples); loss (nullable) row k receives E / 12288 of the start and
// after every step, row stride iters + 1.  The fit's e is only ever set from the accept kernel's reduction, so the history
// cannot increase.  The feature fit's targets come first, the robust fit's automatic scale from the start's x_hat.
int run_lm(ian_handle* h, Plan* pl, const Fit& f, const float* x, float* u, int iters, float* loss, cudaStream_t st) {
  const long long ldl = (long long)iters + 1;
  const bool feats = f.feats();
  auto trial = [&](const float* uu, float* xo) {        // x_hat of uu and, for the feature fit, its features in the planes
    const int r = fit_decode(h, pl, f, uu, xo, st);
    return r != IAN_OK || !feats ? r : run_introspect(h, pl, xo, st);
  };
  int rc;
  if (feats && (rc = feat_targets(h, pl, x, st)) != IAN_OK) return rc;
  if ((rc = trial(u, pl->fxh)) != IAN_OK || (rc = robust_scale(h, f, pl->fxh, x, pl->n, st)) != IAN_OK ||
      (rc = fit_accept(h, pl, f, 1, x, pl->fe, u, loss, ldl, 0, st)) != IAN_OK)
    return rc;
  for (int it = 0; it < iters; ++it) {
    if ((rc = fit_normal_eqs(h, pl, f, u, x, pl->fxh, pl->gnA, pl->gng, pl->gne, st)) != IAN_OK) return rc;
    {
      ScopedTimer tm(h, T_GN_SOLVE, st);
      LAUNCH_TRY(h, launch_gn_solve(pl->gnA, pl->gng, pl->flam, u, pl->fzt, pl->fok, pl->n, st));
    }
    if ((rc = trial(pl->fzt, pl->fxt)) != IAN_OK || (rc = fit_accept(h, pl, f, 0, x, pl->fe, u, loss, ldl, it + 1, st)) != IAN_OK)
      return rc;
  }
  return IAN_OK;
}

// n == 0, the NULL pointers, then for the masked and robust fits the prior weight and, in the host form, every pixel
// weight (the device form cannot read them)
int check_fit_inputs(ian_handle* h, bool host, const Fit& f, int n, const float* w, bool null_ptr) {
  if (n == 0) return IAN_OK;
  if (null_ptr) return fail(h, IAN_ERR_INVALID, "NULL tensor pointer");
  if (f.kind != Fit::MAP && f.kind != Fit::ROBUST) return IAN_OK;
  if (!(f.beta >= 0.0) || !std::isfinite(f.beta))
    return fail(h, IAN_ERR_INVALID, "prior must be finite and >= 0 (got %g)", f.beta);
  if (host && w)
    for (size_t i = 0; i < (size_t)n * 12288; ++i)
      if (!(w[i] >= 0.f) || !std::isfinite(w[i]))
        return fail(h, IAN_ERR_INVALID, "weight %zu (sample %zu) is %g: weights must be finite and >= 0", i, i / 12288, (double)w[i]);
  return IAN_OK;
}

// scale_out (Arg io) of a passed scale: a copy of it
int robust_scale_out(const Chunk& c, const Fit& f, int io) {
  double* o = (double*)c.p[io];
  if (f.kind == Fit::ROBUST && !f.automatic && o && o != f.dl)
    CUDA_TRY(c.h, cudaMemcpyAsync(o, f.dl, (size_t)c.cn * sizeof(double), cudaMemcpyDeviceToDevice, c.st));
  return IAN_OK;
}

// The normal equations at u of every objective (ian_*gauss_newton_*).  No CUDA graphs: the JVP passes run on the 100-row
// plan, whose schedule (stream-K) a capture would change, so both forms launch the same kernels.  The host form stages u
// in the plan's z buffer, x in its image buffer, w in its frame-target buffer, the scales in its scale buffer and A, g, e
// in the plan's own normal-equation buffers.  The robust fit's e comes from robust_accept's reduction (the fit's init form).
int call_normal_eqs(ian_handle* h, bool host, const Fit& fit, const float* u, const float* x, const float* w, const double* scale,
                    int n, double* A, double* g, double* e, double* scale_out, void* stream) {
  int rc = check_fit_inputs(h, host, fit, n, w, !u || !x || !A || !g);
  if (rc != IAN_OK || n == 0) return rc;
  return run_entry(h, host, stream, n, {{u, kLatentBytes, S_Z, IN}, {x, kImageBytes, S_X, IN}, {w, kImageBytes, S_TARGET, IN},
                                        {scale, 8, S_SCALE, IN}, {A, 80000, S_GN_A, OUT}, {g, 800, S_GN_G, OUT},
                                        {e, 8, S_GN_E, OUT}, {scale_out, 8, S_SCALE, OUT}}, kFitPlan[fit.kind],
                   [&](const Chunk& c) {
    Plan* pl = c.pl;
    const Fit f = fit_at(fit, c, 2, 3, 7);
    double* ec = c.p[6] ? (double*)c.p[6] : pl->gne;
    int r = fit_decode(h, pl, f, c.f(0), pl->fxh, c.st);
    if (r == IAN_OK && f.feats() && (r = feat_targets(h, pl, c.f(1), c.st)) == IAN_OK &&
        (r = run_introspect(h, pl, pl->fxh, c.st)) == IAN_OK)
      r = store_features(h, pl, false, nullptr, pl->fcur, 0, c.st);
    if (r == IAN_OK) r = robust_scale(h, f, pl->fxh, c.f(1), c.cn, c.st);
    if (r == IAN_OK) r = fit_normal_eqs(h, pl, f, c.f(0), c.f(1), pl->fxh, (double*)c.p[4], (double*)c.p[5], ec, c.st);
    if (r != IAN_OK || f.kind != Fit::ROBUST) return r;
    if ((r = fit_accept(h, pl, f, 1, c.f(1), ec, c.f(0), nullptr, 1, 0, c.st)) != IAN_OK) return r;
    return robust_scale_out(c, f, 7);
  });
}

// The fit of every objective (ian_fit_latent*_*), in place on u.  The host form stages x in the plan's image buffer, w in
// its frame-target buffer, the scales in its scale buffer, u in its z buffer, z_out in its eps buffer and outlier_w in its
// x_hat buffer, which the fit does not use.  After the fit: rho'(r^2) into outlier_w, z_out = F(u) on the final u, and
// scale_out.
int call_fit(ian_handle* h, bool host, const Fit& fit, const float* x, const float* w, const double* scale, int n, float* u,
             float* z_out, int iters, float* loss, double* scale_out, float* outlier_w, void* stream) {
  int rc = check_fit_inputs(h, host, fit, n, w, !x || !u);
  if (rc != IAN_OK || n == 0) return rc;
  const size_t ldl = (size_t)iters + 1;
  return run_entry(h, host, stream, n, {{x, kImageBytes, S_X, IN}, {w, kImageBytes, S_TARGET, IN}, {scale, 8, S_SCALE, IN},
                                        {u, kLatentBytes, S_Z, INOUT}, {z_out, kLatentBytes, S_EPS, OUT},
                                        {scale_out, 8, S_SCALE, OUT}, {outlier_w, kImageBytes, S_XHAT, OUT}},
                   kFitPlan[fit.kind], [&](const Chunk& c) {
    const Fit f = fit_at(fit, c, 1, 2, 5);
    float* l = nullptr;
    int r = fit_loss_buf(c, loss, ldl, &l);
    if (r == IAN_OK) r = run_lm(h, c.pl, f, c.f(0), c.f(3), iters, l, c.st);
    if (r != IAN_OK) return r;
    if (outlier_w) LAUNCH_TRY(h, launch_robust_outliers(c.pl->fxh, c.f(0), f.w, f.loss, f.dl, c.f(6), c.cn, c.st));
    if (z_out && (r = flow_z(h, c.f(3), c.f(4), nullptr, c.cn, c.st)) != IAN_OK) return r;
    if ((r = robust_scale_out(c, f, 5)) != IAN_OK) return r;
    return fit_loss_out(c, loss, ldl, l);
  });
}

int call_gauss_newton(ian_handle* h, bool host, const float* z, const float* x, int n, double* A, double* g, double* e,
                      void* stream) {
  const int rc = check_fit_args(h, n);
  return rc != IAN_OK ? rc : call_normal_eqs(h, host, Fit{Fit::PLAIN}, z, x, nullptr, nullptr, n, A, g, e, nullptr, stream);
}

int call_fit_latent(ian_handle* h, bool host, const float* x, int n, float* z, int iters, float* loss, void* stream) {
  const int rc = check_fit_args(h, n, iters);
  return rc != IAN_OK ? rc : call_fit(h, host, Fit{Fit::PLAIN}, x, nullptr, nullptr, n, z, nullptr, iters, loss, nullptr,
                                      nullptr, stream);
}

int call_map_gauss_newton(ian_handle* h, bool host, const float* u, const float* x, const float* w, double prior, int n,
                          double* A, double* g, double* e, void* stream) {
  const int rc = check_fit_args(h, n);
  return rc != IAN_OK ? rc : call_normal_eqs(h, host, Fit{Fit::MAP, has_flow(h), prior}, u, x, w, nullptr, n, A, g, e,
                                             nullptr, stream);
}

int call_fit_latent_map(ian_handle* h, bool host, const float* x, const float* w, double prior, int n, float* u, float* z_out,
                        int iters, float* loss, void* stream) {
  const int rc = check_fit_args(h, n, iters);
  return rc != IAN_OK ? rc : call_fit(h, host, Fit{Fit::MAP, has_flow(h), prior}, x, w, nullptr, n, u, z_out, iters, loss,
                                      nullptr, nullptr, stream);
}

int call_robust_gauss_newton(ian_handle* h, bool host, const float* u, const float* x, const float* w, double prior, int kind,
                             const double* scale, int n, double* A, double* g, double* e, double* scale_out, void* stream) {
  int rc = check_fit_args(h, n);
  if (rc != IAN_OK || (rc = check_robust_args(h, host, n, kind, scale)) != IAN_OK) return rc;
  return call_normal_eqs(h, host, Fit{Fit::ROBUST, has_flow(h), prior, kind}, u, x, w, scale, n, A, g, e, scale_out, stream);
}

int call_fit_latent_robust(ian_handle* h, bool host, const float* x, const float* w, double prior, int kind, const double* scale,
                           int n, float* u, float* z_out, int iters, float* loss, double* scale_out, float* outlier_w,
                           void* stream) {
  int rc = check_fit_args(h, n, iters);
  if (rc != IAN_OK || (rc = check_robust_args(h, host, n, kind, scale)) != IAN_OK) return rc;
  return call_fit(h, host, Fit{Fit::ROBUST, has_flow(h), prior, kind}, x, w, scale, n, u, z_out, iters, loss, scale_out,
                  outlier_w, stream);
}

int call_feature_gauss_newton(ian_handle* h, bool host, const float* z, const float* x, int n, double a, double b, double* A,
                              double* g, double* e, void* stream) {
  int rc = check_fit_args(h, n);
  if (rc != IAN_OK || (rc = check_feat_weights(h, a, b)) != IAN_OK) return rc;
  return call_normal_eqs(h, host, feature_fit(a, b), z, x, nullptr, nullptr, n, A, g, e, nullptr, stream);
}

int call_fit_latent_features(ian_handle* h, bool host, const float* x, int n, float* z, int iters, double a, double b, float* loss,
                             void* stream) {
  int rc = check_fit_args(h, n, iters);
  if (rc != IAN_OK || (rc = check_feat_weights(h, a, b)) != IAN_OK) return rc;
  return call_fit(h, host, feature_fit(a, b), x, nullptr, nullptr, n, z, nullptr, iters, loss, nullptr, nullptr, stream);
}

}  // namespace

// ================================================================================================
// C-ABI
// ================================================================================================
extern "C" {

int ian_create(int model_kind, int device, ian_handle** out) {
  if (!out) return fail(nullptr, IAN_ERR_INVALID, "out is NULL");
  if (model_kind != IAN_MODEL_SIMPLE && model_kind != IAN_MODEL_FULL && model_kind != IAN_MODEL_V1)
    return fail(nullptr, IAN_ERR_UNSUPPORTED, "unknown model kind %d", model_kind);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(nullptr, IAN_ERR_CUDA, "no CUDA device: %s (this library has no CPU path)", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(nullptr, IAN_ERR_INVALID, "device %d out of range [0,%d)", device, ndev);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, IAN_ERR_UNSUPPORTED, "device %d is sm_%d%d; libian_b200 is built for sm_90a only", device, prop.major, prop.minor);
  ian_handle* h = new ian_handle();
  h->device = device;
  h->model_kind = model_kind;
  DeviceGuard dg(device);
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->h2d_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->d2h_stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete h;
    return fail(nullptr, IAN_ERR_CUDA, "cudaStreamCreate failed");
  }
  if (const char* c = getenv("IAN_CHUNK")) { int v = atoi(c); if (v > 0) h->max_chunk = v > 4096 ? 4096 : v; }
  if (const char* c = getenv("IAN_PATH")) { if (!strcmp(c, "simt")) h->path = IAN_PATH_SIMT; }
  if (const char* c = getenv("IAN_STREAMK")) { const int v = atoi(c); h->streamk = v < 0 ? 0 : v > 2 ? 2 : v; }
  if (const char* c = getenv("IAN_SPLITK")) h->splitk = atoi(c) != 0;
  if (const char* c = getenv("IAN_PDL")) h->pdl = atoi(c) != 0;
  if (const char* c = getenv("IAN_FINALIZE8")) h->coop_finalize = atoi(c) != 0;
  if (const char* c = getenv("IAN_GRAPHS")) h->graphs = atoi(c) != 0;
  if (const char* c = getenv("IAN_EPI_TMA")) h->epi_tma = atoi(c) != 0;
  *out = h;
  return IAN_OK;
}

int ian_set_param(ian_handle* h, const char* name, const float* data, const int64_t* shape, int ndim) {
  if (!h || !name || !data || !shape) return fail(h, IAN_ERR_INVALID, "NULL argument");
  if (h->finalized) return fail(h, IAN_ERR_STATE, "model already finalized");
  int64_t elems = 0;
  int rc = check_param_shape(h, name, shape, ndim, &elems);
  if (rc != IAN_OK) return rc;
  HostParam& p = h->params[name];
  p.shape.assign(shape, shape + ndim);
  p.data.assign(data, data + elems);
  return IAN_OK;
}

int ian_set_made_ordering(ian_handle* h, const int32_t* ordering, int n) {
  if (!h || !ordering) return fail(h, IAN_ERR_INVALID, "NULL argument");
  if (h->finalized) return fail(h, IAN_ERR_STATE, "model already finalized");
  if (n != 100) return fail(h, IAN_ERR_INVALID, "ordering must have 100 entries (got %d)", n);
  std::vector<char> seen(100, 0);
  for (int i = 0; i < n; ++i) {
    if (ordering[i] < 0 || ordering[i] >= 100 || seen[ordering[i]]) return fail(h, IAN_ERR_INVALID, "ordering is not a permutation of 0..99");
    seen[ordering[i]] = 1;
  }
  h->made_ordering.assign(ordering, ordering + n);
  return IAN_OK;
}

// The model's OWN parameter list: what `lasagne.layers.get_all_params(...)` hands GANcheckpoints.load_weights in the
// reference (API.py:23-30).  A loader iterates these names and looks each one up in the checkpoint, so that extra keys
// of the file (log_sigma_theta, discriminator weights, metadata ...) are ignored exactly as the reference does.
int ian_model_param_count(int model_kind) {
  if (model_kind < 0 || model_kind > 2) return IAN_ERR_INVALID;
  return (int)cached_specs(model_kind).size();
}

int ian_model_param_spec(int model_kind, int index, const char** name, int64_t* shape /*[4]*/, int* ndim) {
  if (model_kind < 0 || model_kind > 2 || !name || !shape || !ndim) return IAN_ERR_INVALID;
  const auto& v = cached_specs(model_kind);
  if (index < 0 || index >= (int)v.size()) return IAN_ERR_INVALID;
  *name = v[index].name.c_str();
  *ndim = (int)v[index].shape.size();
  for (int i = 0; i < 4; ++i) shape[i] = i < *ndim ? v[index].shape[i] : 1;
  return IAN_OK;
}

int ian_made_mask(const int32_t* ordering, int n, int which, uint8_t* mask_out /*[100][100], (in,out)*/) {
  if (!ordering || !mask_out || n != 100 || which < 0 || which > 2) return IAN_ERR_INVALID;
  for (int i = 0; i < 100; ++i)
    for (int j = 0; j < 100; ++j) mask_out[i * 100 + j] = made_keep(ordering, which, i, j) ? 1 : 0;
  return IAN_OK;
}

int ian_debug_made_weights(ian_handle* h, float* out /*[2][3][100][100]*/) {
  if (!h || !out) return IAN_ERR_INVALID;
  if (!h->finalized || !h->made_w) return fail(h, IAN_ERR_STATE, "no MADE weights on this handle (IAN_simple, or not finalized)");
  DeviceGuard dg(h->device);
  CUDA_TRY(h, cudaMemcpy(out, h->made_w, (size_t)2 * 3 * 10000 * sizeof(float), cudaMemcpyDeviceToHost));
  return IAN_OK;
}

int ian_finalize(ian_handle* h) {
  if (!h) return IAN_ERR_INVALID;
  if (h->finalized) return IAN_OK;
  for (const auto& sp : cached_specs(h->model_kind))
    if (!h->params.count(sp.name)) return fail(h, IAN_ERR_STATE, "missing parameter '%s'", sp.name.c_str());
  DeviceGuard dg(h->device);
  int rc = prepare_encoder(h);
  if (rc != IAN_OK) return rc;
  rc = h->model_kind == IAN_MODEL_FULL ? prepare_full_decoder(h)
       : h->model_kind == IAN_MODEL_V1 ? prepare_v1_decoder(h) : prepare_simple_decoder(h);
  if (rc != IAN_OK) return rc;
  CUDA_TRY(h, cudaMalloc((void**)&h->sk_ws, tc_sk_workspace_floats() * sizeof(float)));
  CUDA_TRY(h, cudaMalloc((void**)&h->sk_flags, tc_sk_flag_ints() * sizeof(int)));
  CUDA_TRY(h, cudaMemset(h->sk_flags, 0, tc_sk_flag_ints() * sizeof(int)));
  h->params.clear();
  h->finalized = true;
  return IAN_OK;
}

int ian_destroy(ian_handle* h) {
  if (!h) return IAN_OK;
  DeviceGuard dg(h->device);
  cudaStreamSynchronize(h->stream);
  cudaStreamSynchronize(h->h2d_stream);
  cudaStreamSynchronize(h->d2h_stream);
  for (auto& kv : h->plans) free_plan(kv.second);
  for (auto& w : h->w) { cudaFree(w.b); cudaFree(w.scale); cudaFree(w.shift); }
  cudaFree(h->conv1_wt); cudaFree(h->conv1_b); cudaFree(h->decout_wt); cudaFree(h->decout_tc_wt); cudaFree(h->conv1_bwd_wt); cudaFree(h->conv1_bwd_tc_wt);
  cudaFree(h->sk_ws); cudaFree(h->sk_flags);
  for (auto& s : h->dec_bn_stats) { cudaFree(s[0]); cudaFree(s[1]); }
  for (float* p : h->pv_dev) cudaFree(p);
  cudaFree(h->conv1_tc_wt); if (h->conv1_maps) conv1_free_maps(h->conv1_maps);
  cudaFree(h->made_w); cudaFree(h->made_b); cudaFree(h->head_taps); cudaFree(h->head_wgb); cudaFree(h->head_wbb);
  cudaFree(h->head_tc_wt);
  cudaFree(h->train_ws);
  cudaFree(h->gn_eye); cudaFree(h->gn_zrep); cudaFree(h->gn_J); cudaFree(h->gn_part); cudaFree(h->map_flow); cudaFree(h->feat_part);
  for (float* p : h->disc_w) cudaFree(p);
  cudaFree(h->disc_buf);
  cudaFree(h->enc_bn_gb);
  cudaFree(h->dec_bn_gb);
  for (auto& s : h->bn_bufs) cudaFree(s.buf);
  for (auto& v : h->timed) for (auto& t : v) { cudaEventDestroy(t.e0); cudaEventDestroy(t.e1); }
  if (h->push_stream) { cudaStreamSynchronize(h->push_stream); cudaStreamDestroy(h->push_stream); }
  for (int b = 0; b < 2; ++b) { if (h->g_comp[b]) cudaEventDestroy(h->g_comp[b]); if (h->g_done[b]) cudaEventDestroy(h->g_done[b]); }
  for (int r = 0; r < h->gw; ++r) if (r != h->grank && h->gpeer_buf[r]) cudaIpcCloseMemHandle(h->gpeer_buf[r]);
  cudaFree(h->gbuf);
  for (void* p : h->host_allocs) cudaFreeHost(p);
  cudaStreamDestroy(h->stream);
  cudaStreamDestroy(h->h2d_stream);
  cudaStreamDestroy(h->d2h_stream);
  delete h;
  return IAN_OK;
}

const char* ian_last_error(const ian_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }
int ian_get_zdim(const ian_handle*) { return 100; }
int64_t ian_launch_count(const ian_handle* h) { return h ? h->launches : 0; }

int ian_set_path(ian_handle* h, int path) {
  if (!h) return IAN_ERR_INVALID;
  if (path != IAN_PATH_TC && path != IAN_PATH_SIMT) return fail(h, IAN_ERR_INVALID, "unknown path %d", path);
  h->path = path;
  return IAN_OK;
}

int ian_set_precision(ian_handle* h, int precision) {
  if (!h) return IAN_ERR_INVALID;
  if (precision != IAN_PRECISION_FP32 && precision != IAN_PRECISION_BF16) return fail(h, IAN_ERR_INVALID, "unknown precision %d", precision);
  if (precision == IAN_PRECISION_BF16 && h->model_kind == IAN_MODEL_SIMPLE)
    return fail(h, IAN_ERR_UNSUPPORTED, "bf16 mode is built for the IAN.py / IANv1.py graphs (BASELINE configs[2]); IAN_simple runs in float32");
  h->passes = precision == IAN_PRECISION_BF16 ? 1 : 3;
  return IAN_OK;
}

int ian_set_layer_timing(ian_handle* h, int enable) {
  if (!h) return IAN_ERR_INVALID;
  h->timing = enable != 0;
  return IAN_OK;
}

double ian_layer_time_ms(ian_handle* h, const char* layer_name, int reset) {
  if (!h || !layer_name) return -1.0;
  DeviceGuard dg(h->device);
  for (int l = 0; l < T_COUNT; ++l) {
    if (strcmp(kLayerNames[l], layer_name)) continue;
    for (auto& t : h->timed[l]) {
      float ms = 0.f;
      if (cudaEventSynchronize(t.e1) == cudaSuccess && cudaEventElapsedTime(&ms, t.e0, t.e1) == cudaSuccess) {
        h->time_ms[l] += ms;
        h->time_cnt[l] += 1;
      }
      cudaEventDestroy(t.e0);
      cudaEventDestroy(t.e1);
    }
    h->timed[l].clear();
    const double r = h->time_cnt[l] ? h->time_ms[l] / (double)h->time_cnt[l] : -1.0;
    if (reset) { h->time_ms[l] = 0; h->time_cnt[l] = 0; }
    return r;
  }
  return -1.0;
}

// Replace one IAN_simple decoder parameter of a finalized handle: re-derive what ian_finalize derives from its group and
// write it into the same device buffers (tiles of both directions, dec_out's two weight forms, folded BatchNorm vectors).
// The device is synchronised first, so the update is ordered after all work enqueued before the call.
int ian_update_param_host(ian_handle* h, const char* name, const float* data, const int64_t* shape, int ndim) {
  if (!h || !name || !data || !shape) return fail(h, IAN_ERR_INVALID, "NULL argument");
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "the handle is not finalized: use ian_set_param");
  if (h->model_kind != IAN_MODEL_SIMPLE) return fail(h, IAN_ERR_UNSUPPORTED, "in-place updates are implemented for IAN_simple only");
  const std::string n(name);
  int group = -1, bn = -1, field = -1;                 // group: 0 fc2, 1..3 dec_conv, 4 dec_out, 5 BatchNorm
  if (n == "l_dec_fc2.W") group = 0;
  for (int k = 0; k < 3; ++k) if (n == kDecConv[k].w) group = 1 + k;
  if (n == "dec_out.W") group = 4;
  for (int k = 0; k < 4; ++k)
    for (int f = 0; f < 4; ++f)
      if (n == std::string(kDecBn[k]) + "." + kBnFields[f]) { group = 5; bn = k; field = f; }
  if (group < 0) return fail(h, IAN_ERR_INVALID, "'%s' is not an IAN_simple decoder parameter that can be updated", name);
  int64_t elems = 0;
  int rc = check_param_shape(h, name, shape, ndim, &elems);
  if (rc != IAN_OK) return rc;
  DeviceGuard dg(h->device);
  CUDA_TRY(h, cudaDeviceSynchronize());
  const std::vector<float> v(data, data + elems);
  if (group == 0) return simple_fc2_weights(h, v);
  if (group <= 3) return simple_conv_weights(h, group - 1, v);
  if (group == 4) return simple_dec_out_weights(h, v);
  h->dec_bn[bn][field] = v;
  return simple_bn(h, bn);
}

// ---- batch entry points: one body each (call_*), in the device and the host form ---------------------------------
int ian_encode_dev(ian_handle* h, const float* x, int n, const float* eps, float* z, void* stream) {
  return call_encode(h, false, x, n, eps, z, stream);
}
int ian_encode_host(ian_handle* h, const float* x, int n, const float* eps, float* z) {
  return call_encode(h, true, x, n, eps, z, nullptr);
}

int ian_decode_dev(ian_handle* h, const float* z, int n, float* x, void* stream) { return call_decode(h, false, z, n, x, stream); }
int ian_decode_host(ian_handle* h, const float* z, int n, float* x) { return call_decode(h, true, z, n, x, nullptr); }

int ian_reconstruct_dev(ian_handle* h, const float* x, int n, float* z_out, float* x_hat, void* stream) {
  return call_reconstruct(h, false, x, n, z_out, x_hat, stream);
}
int ian_reconstruct_host(ian_handle* h, const float* x, int n, float* z_out, float* x_hat) {
  return call_reconstruct(h, true, x, n, z_out, x_hat, nullptr);
}

int ian_grad_dev(ian_handle* h, const float* z, const int32_t* boxes, const float* target, int target_is_frame, int n,
                 float* g, void* stream) {
  return call_grad(h, false, z, boxes, target, target_is_frame, n, g, stream);
}
int ian_grad_host(ian_handle* h, const float* z, const int32_t* boxes, const float* target, int target_is_frame, int n,
                  float* g) {
  return call_grad(h, true, z, boxes, target, target_is_frame, n, g, nullptr);
}

int ian_decode_vjp_dev(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz, void* stream) {
  return call_decode_vjp(h, false, z, dx_hat, n, dz, stream);
}
int ian_decode_vjp_host(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz) {
  return call_decode_vjp(h, true, z, dx_hat, n, dz, nullptr);
}
int ian_decode_jvp_dev(ian_handle* h, const float* z, const float* v, int n, float* x_hat, float* dx_hat, void* stream) {
  return call_decode_jvp(h, false, z, v, n, x_hat, dx_hat, stream);
}
int ian_decode_jvp_host(ian_handle* h, const float* z, const float* v, int n, float* x_hat, float* dx_hat) {
  return call_decode_jvp(h, true, z, v, n, x_hat, dx_hat, nullptr);
}
int ian_encode_jvp_dev(ian_handle* h, const float* x, const float* v, int n, const float* eps, float* z, float* dz, void* stream) {
  return call_encode_jvp(h, false, x, v, n, eps, z, dz, stream);
}
int ian_encode_jvp_host(ian_handle* h, const float* x, const float* v, int n, const float* eps, float* z, float* dz) {
  return call_encode_jvp(h, true, x, v, n, eps, z, dz, nullptr);
}

int ian_param_vjp_supported(int model_kind, int index) { return pv_slot(model_kind, index) >= 0 ? 1 : 0; }
int ian_decode_param_vjp_dev(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz, float* const* grads,
                             void* stream) {
  return call_param_vjp(h, false, z, dx_hat, n, dz, grads, stream);
}
int ian_decode_param_vjp_host(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz, float* const* grads) {
  return call_param_vjp(h, true, z, dx_hat, n, dz, grads, nullptr);
}

int ian_encode_vjp_dev(ian_handle* h, const float* x, int n, const float* eps, const float* dz, float* dx, void* stream) {
  return call_encode_vjp(h, false, x, n, eps, dz, dx, stream);
}
int ian_encode_vjp_host(ian_handle* h, const float* x, int n, const float* eps, const float* dz, float* dx) {
  return call_encode_vjp(h, true, x, n, eps, dz, dx, nullptr);
}

int ian_decode_gauss_newton_dev(ian_handle* h, const float* z, const float* x, int n, double* A, double* g, double* e,
                                void* stream) {
  return call_gauss_newton(h, false, z, x, n, A, g, e, stream);
}
int ian_decode_gauss_newton_host(ian_handle* h, const float* z, const float* x, int n, double* A, double* g, double* e) {
  return call_gauss_newton(h, true, z, x, n, A, g, e, nullptr);
}
int ian_fit_latent_dev(ian_handle* h, const float* x, int n, float* z, int iters, float* loss, void* stream) {
  return call_fit_latent(h, false, x, n, z, iters, loss, stream);
}
int ian_fit_latent_host(ian_handle* h, const float* x, int n, float* z, int iters, float* loss) {
  return call_fit_latent(h, true, x, n, z, iters, loss, nullptr);
}
int ian_map_gauss_newton_dev(ian_handle* h, const float* u, const float* x, const float* w, double prior, int n, double* A,
                             double* g, double* e, void* stream) {
  return call_map_gauss_newton(h, false, u, x, w, prior, n, A, g, e, stream);
}
int ian_map_gauss_newton_host(ian_handle* h, const float* u, const float* x, const float* w, double prior, int n, double* A,
                              double* g, double* e) {
  return call_map_gauss_newton(h, true, u, x, w, prior, n, A, g, e, nullptr);
}
int ian_fit_latent_map_dev(ian_handle* h, const float* x, const float* w, double prior, int n, float* u, float* z_out, int iters,
                           float* loss, void* stream) {
  return call_fit_latent_map(h, false, x, w, prior, n, u, z_out, iters, loss, stream);
}
int ian_fit_latent_map_host(ian_handle* h, const float* x, const float* w, double prior, int n, float* u, float* z_out, int iters,
                            float* loss) {
  return call_fit_latent_map(h, true, x, w, prior, n, u, z_out, iters, loss, nullptr);
}

int ian_robust_gauss_newton_dev(ian_handle* h, const float* u, const float* x, const float* w, double prior, int kind,
                                const double* scale, int n, double* A, double* g, double* e, double* scale_out, void* stream) {
  return call_robust_gauss_newton(h, false, u, x, w, prior, kind, scale, n, A, g, e, scale_out, stream);
}
int ian_robust_gauss_newton_host(ian_handle* h, const float* u, const float* x, const float* w, double prior, int kind,
                                 const double* scale, int n, double* A, double* g, double* e, double* scale_out) {
  return call_robust_gauss_newton(h, true, u, x, w, prior, kind, scale, n, A, g, e, scale_out, nullptr);
}
int ian_fit_latent_robust_dev(ian_handle* h, const float* x, const float* w, double prior, int kind, const double* scale, int n,
                              float* u, float* z_out, int iters, float* loss, double* scale_out, float* outlier_w, void* stream) {
  return call_fit_latent_robust(h, false, x, w, prior, kind, scale, n, u, z_out, iters, loss, scale_out, outlier_w, stream);
}
int ian_fit_latent_robust_host(ian_handle* h, const float* x, const float* w, double prior, int kind, const double* scale, int n,
                               float* u, float* z_out, int iters, float* loss, double* scale_out, float* outlier_w) {
  return call_fit_latent_robust(h, true, x, w, prior, kind, scale, n, u, z_out, iters, loss, scale_out, outlier_w, nullptr);
}

int ian_introspect_dev(ian_handle* h, const float* x, int n, float* f1, float* f2, float* f3, float* f4, void* stream) {
  float* f[4] = {f1, f2, f3, f4};
  return call_introspect(h, false, x, n, f, stream);
}
int ian_introspect_host(ian_handle* h, const float* x, int n, float* f1, float* f2, float* f3, float* f4) {
  float* f[4] = {f1, f2, f3, f4};
  return call_introspect(h, true, x, n, f, nullptr);
}
int ian_introspect_jvp_dev(ian_handle* h, const float* x, const float* v, int n, float* f1, float* f2, float* f3, float* f4,
                           float* t1, float* t2, float* t3, float* t4, void* stream) {
  float* f[4] = {f1, f2, f3, f4};
  float* t[4] = {t1, t2, t3, t4};
  return call_introspect_jvp(h, false, x, v, n, f, t, stream);
}
int ian_introspect_jvp_host(ian_handle* h, const float* x, const float* v, int n, float* f1, float* f2, float* f3, float* f4,
                            float* t1, float* t2, float* t3, float* t4) {
  float* f[4] = {f1, f2, f3, f4};
  float* t[4] = {t1, t2, t3, t4};
  return call_introspect_jvp(h, true, x, v, n, f, t, nullptr);
}
int ian_introspect_vjp_dev(ian_handle* h, const float* x, int n, const float* c1, const float* c2, const float* c3,
                           const float* c4, float* dx, void* stream) {
  const float* c[4] = {c1, c2, c3, c4};
  return call_introspect_vjp(h, false, x, n, c, dx, stream);
}
int ian_introspect_vjp_host(ian_handle* h, const float* x, int n, const float* c1, const float* c2, const float* c3,
                            const float* c4, float* dx) {
  const float* c[4] = {c1, c2, c3, c4};
  return call_introspect_vjp(h, true, x, n, c, dx, nullptr);
}
int ian_set_discriminator_param(ian_handle* h, const char* name, const float* data, const int64_t* shape, int ndim) {
  if (!h) return IAN_ERR_INVALID;
  if (!name || !data || !shape) return fail(h, IAN_ERR_INVALID, "NULL argument");
  int k = 0;
  while (k < 4 && strcmp(name, kDiscParams[k])) ++k;
  if (k == 4) return fail(h, IAN_ERR_INVALID, "'%s' is not a discriminator parameter", name);
  const int64_t want[4][3] = {{1024, kDiscKernels, kDiscDims}, {kDiscKernels, kDiscDims}, {kDiscKernels}, {kDiscIn, disc_units(h)}};
  const int nd[4] = {3, 2, 1, 2};
  bool ok = ndim == nd[k];
  int64_t elems = 1;
  for (int i = 0; ok && i < ndim; ++i) {
    ok = shape[i] == want[k][i];
    elems *= want[k][i];
  }
  if (!ok) return fail(h, IAN_ERR_INVALID, "'%s' has the wrong shape (want %d dims: %lld %lld %lld)", name, nd[k],
                       (long long)want[k][0], (long long)want[k][1], (long long)want[k][2]);
  DeviceGuard dg(h->device);
  if (h->disc_w[k]) CUDA_TRY(h, cudaDeviceSynchronize());   // ordered after all work enqueued before the call
  else CUDA_TRY(h, cudaMalloc((void**)&h->disc_w[k], (size_t)elems * sizeof(float)));
  CUDA_TRY(h, cudaMemcpy(h->disc_w[k], data, (size_t)elems * sizeof(float), cudaMemcpyHostToDevice));
  h->disc_set |= 1 << k;
  return IAN_OK;
}
int ian_discriminate_dev(ian_handle* h, const float* x, int n, float* logits, float* p, void* stream) {
  return call_discriminate(h, false, x, n, logits, p, stream);
}
int ian_discriminate_host(ian_handle* h, const float* x, int n, float* logits, float* p) {
  return call_discriminate(h, true, x, n, logits, p, nullptr);
}
int ian_discriminate_vjp_dev(ian_handle* h, const float* x, int n, const float* dlogits, float* dx, void* stream) {
  return call_discriminate_vjp(h, false, x, n, dlogits, dx, stream);
}
int ian_discriminate_vjp_host(ian_handle* h, const float* x, int n, const float* dlogits, float* dx) {
  return call_discriminate_vjp(h, true, x, n, dlogits, dx, nullptr);
}
int ian_discriminate_train_dev(ian_handle* h, const float* x, int n, float* logits, float* p, float* stats, void* stream) {
  return call_discriminate_train(h, false, x, n, logits, p, stats, stream);
}
int ian_discriminate_train_host(ian_handle* h, const float* x, int n, float* logits, float* p, float* stats) {
  return call_discriminate_train(h, true, x, n, logits, p, stats, nullptr);
}
int ian_discriminate_train_vjp_dev(ian_handle* h, const float* x, int n, const float* dlogits, float* dx, void* stream) {
  return call_discriminate_train_vjp(h, false, x, n, dlogits, dx, stream);
}
int ian_discriminate_train_vjp_host(ian_handle* h, const float* x, int n, const float* dlogits, float* dx) {
  return call_discriminate_train_vjp(h, true, x, n, dlogits, dx, nullptr);
}
int ian_decode_train_dev(ian_handle* h, const float* z, int n, float* x_hat, float* stats, void* stream) {
  return call_decode_train(h, false, z, n, x_hat, stats, stream);
}
int ian_decode_train_host(ian_handle* h, const float* z, int n, float* x_hat, float* stats) {
  return call_decode_train(h, true, z, n, x_hat, stats, nullptr);
}
int ian_decode_train_vjp_dev(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz, float* const* grads,
                             void* stream) {
  return call_decode_train_vjp(h, false, z, dx_hat, n, dz, grads, stream);
}
int ian_decode_train_vjp_host(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz, float* const* grads) {
  return call_decode_train_vjp(h, true, z, dx_hat, n, dz, grads, nullptr);
}
int ian_feature_gauss_newton_dev(ian_handle* h, const float* z, const float* x, int n, double pixel_weight, double feature_weight,
                                 double* A, double* g, double* e, void* stream) {
  return call_feature_gauss_newton(h, false, z, x, n, pixel_weight, feature_weight, A, g, e, stream);
}
int ian_feature_gauss_newton_host(ian_handle* h, const float* z, const float* x, int n, double pixel_weight,
                                  double feature_weight, double* A, double* g, double* e) {
  return call_feature_gauss_newton(h, true, z, x, n, pixel_weight, feature_weight, A, g, e, nullptr);
}
int ian_fit_latent_features_dev(ian_handle* h, const float* x, int n, float* z, int iters, double pixel_weight,
                                double feature_weight, float* loss, void* stream) {
  return call_fit_latent_features(h, false, x, n, z, iters, pixel_weight, feature_weight, loss, stream);
}
int ian_fit_latent_features_host(ian_handle* h, const float* x, int n, float* z, int iters, double pixel_weight,
                                 double feature_weight, float* loss) {
  return call_fit_latent_features(h, true, x, n, z, iters, pixel_weight, feature_weight, loss, nullptr);
}

int ian_edit_loop_dev(ian_handle* h, float* z, const int32_t* boxes, const float* target, int target_is_frame, int n,
                      int n_steps, float weight, void* stream) {
  return call_edit_loop(h, false, z, boxes, target, target_is_frame, n, n_steps, weight, stream);
}
int ian_edit_loop_host(ian_handle* h, float* z, const int32_t* boxes, const float* target, int target_is_frame, int n,
                       int n_steps, float weight) {
  return call_edit_loop(h, true, z, boxes, target, target_is_frame, n, n_steps, weight, nullptr);
}

// ---- pipelined host API -----------------------------------------------------------------------------
int ian_host_alloc(ian_handle* h, size_t bytes, void** out) {
  if (!h || !out || bytes == 0) return fail(h, IAN_ERR_INVALID, "bad argument");
  DeviceGuard dg(h->device);
  void* p = nullptr;
  CUDA_TRY(h, cudaHostAlloc(&p, bytes, cudaHostAllocDefault));
  h->host_allocs.push_back(p);
  *out = p;
  return IAN_OK;
}

int ian_host_free(ian_handle* h, void* p) {
  if (!h || !p) return IAN_ERR_INVALID;
  for (size_t i = 0; i < h->host_allocs.size(); ++i)
    if (h->host_allocs[i] == p) {
      h->host_allocs.erase(h->host_allocs.begin() + i);
      DeviceGuard dg(h->device);
      CUDA_TRY(h, cudaFreeHost(p));
      return IAN_OK;
    }
  return fail(h, IAN_ERR_INVALID, "pointer was not allocated by ian_host_alloc");
}

int ian_reconstruct_submit(ian_handle* h, const float* x, int n, float* z_out, float* x_hat, int* ticket) {
  int rc = check_ready(h, n, x, x_hat);
  if (rc != IAN_OK) return rc;
  if (!ticket) return fail(h, IAN_ERR_INVALID, "ticket is NULL");
  if (n > h->max_chunk) return fail(h, IAN_ERR_INVALID, "pipelined calls take at most %d images (got %d)", h->max_chunk, n);
  DeviceGuard dg(h->device);
  Plan* pl = nullptr;
  if ((rc = get_plan(h, n, &pl)) != IAN_OK) return rc;
  const int s = (int)(h->tickets & 1);
  if (h->inflight[s].id >= 0) {                          // the request that used this slot two submits ago (any plan) is done
    auto prev = h->plans.find(h->inflight[s].n);
    if (prev != h->plans.end() && prev->second->ev_d2h[s]) CUDA_TRY(h, cudaEventSynchronize(prev->second->ev_d2h[s]));
  }
  if (!pl->sx[s]) {
    for (int b = 0; b < 2; ++b) {
      if ((rc = alloc_buf(h, pl, pl->sx[b], (long long)n * 12288)) != IAN_OK) return rc;
      if ((rc = alloc_buf(h, pl, pl->sz[b], (long long)n * 100)) != IAN_OK) return rc;
      if ((rc = alloc_buf(h, pl, pl->sxh[b], (long long)n * 12288)) != IAN_OK) return rc;
      CUDA_TRY(h, cudaEventCreateWithFlags(&pl->ev_h2d[b], cudaEventDisableTiming));
      CUDA_TRY(h, cudaEventCreateWithFlags(&pl->ev_comp[b], cudaEventDisableTiming));
      CUDA_TRY(h, cudaEventCreateWithFlags(&pl->ev_d2h[b], cudaEventDisableTiming));
    }
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));     // the memsets of the new buffers
  }
  CUDA_TRY(h, cudaMemcpyAsync(pl->sx[s], x, (size_t)n * 12288 * 4, cudaMemcpyHostToDevice, h->h2d_stream));
  CUDA_TRY(h, cudaEventRecord(pl->ev_h2d[s], h->h2d_stream));
  CUDA_TRY(h, cudaStreamWaitEvent(h->stream, pl->ev_h2d[s], 0));
  if ((rc = run_encode(h, pl, pl->sx[s], nullptr, pl->sz[s], h->stream)) != IAN_OK) return rc;
  if ((rc = run_decode_from_planes(h, pl, pl->sxh[s], h->stream)) != IAN_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(pl->ev_comp[s], h->stream));
  CUDA_TRY(h, cudaStreamWaitEvent(h->d2h_stream, pl->ev_comp[s], 0));
  CUDA_TRY(h, cudaMemcpyAsync(x_hat, pl->sxh[s], (size_t)n * 12288 * 4, cudaMemcpyDeviceToHost, h->d2h_stream));
  if (z_out) CUDA_TRY(h, cudaMemcpyAsync(z_out, pl->sz[s], (size_t)n * 400, cudaMemcpyDeviceToHost, h->d2h_stream));
  CUDA_TRY(h, cudaEventRecord(pl->ev_d2h[s], h->d2h_stream));
  const int id = (int)(h->tickets & 0x7fffffff);             // monotonically increasing; mapped to (plan, slot) below
  h->inflight[s].id = id; h->inflight[s].n = n; h->inflight[s].slot = s;
  *ticket = id;
  h->tickets += 1;
  return IAN_OK;
}

int ian_reconstruct_wait(ian_handle* h, int ticket) {
  if (!h) return IAN_ERR_INVALID;
  if (ticket < 0 || (long long)ticket >= h->tickets) return fail(h, IAN_ERR_INVALID, "unknown ticket %d", ticket);
  const ian_handle::Ticket* tk = nullptr;
  for (const auto& t : h->inflight) if (t.id == ticket) tk = &t;
  if (!tk) return IAN_OK;      // older than the two requests in flight: its slot was reused, i.e. it completed (submit waited)
  auto it = h->plans.find(tk->n);
  if (it == h->plans.end() || !it->second->ev_d2h[tk->slot]) return fail(h, IAN_ERR_INVALID, "unknown ticket %d", ticket);
  DeviceGuard dg(h->device);
  CUDA_TRY(h, cudaEventSynchronize(it->second->ev_d2h[tk->slot]));
  return IAN_OK;
}

// ---- sample_IAN.py function set (reference sample_IAN.py:86-94) and its derivatives ---------------------------------------
int ian_encode_pre_dev(ian_handle* h, const float* x, int n, float* z_iaf, void* stream) {
  return call_encode_pre(h, false, x, n, z_iaf, stream);
}
int ian_encode_pre_host(ian_handle* h, const float* x, int n, float* z_iaf) {
  return call_encode_pre(h, true, x, n, z_iaf, nullptr);
}
int ian_flow_dev(ian_handle* h, const float* z_iaf, int n, float* z_out, float* x_out, void* stream) {
  return call_flow(h, false, z_iaf, n, z_out, x_out, stream);
}
int ian_flow_host(ian_handle* h, const float* z_iaf, int n, float* z_out, float* x_out) {
  return call_flow(h, true, z_iaf, n, z_out, x_out, nullptr);
}
int ian_flow_vjp_dev(ian_handle* h, const float* z_iaf, const float* dz, int n, float* dz_iaf, void* stream) {
  return call_flow_vjp(h, false, z_iaf, dz, n, dz_iaf, stream);
}
int ian_flow_vjp_host(ian_handle* h, const float* z_iaf, const float* dz, int n, float* dz_iaf) {
  return call_flow_vjp(h, true, z_iaf, dz, n, dz_iaf, nullptr);
}
int ian_flow_jvp_dev(ian_handle* h, const float* z_iaf, const float* v, int n, float* z, float* dz, void* stream) {
  return call_flow_jvp(h, false, z_iaf, v, n, z, dz, stream);
}
int ian_flow_jvp_host(ian_handle* h, const float* z_iaf, const float* v, int n, float* z, float* dz) {
  return call_flow_jvp(h, true, z_iaf, v, n, z, dz, nullptr);
}
int ian_encode_pre_vjp_dev(ian_handle* h, const float* x, int n, const float* dz_iaf, float* dx, void* stream) {
  return call_encode_pre_vjp(h, false, x, n, dz_iaf, dx, stream);
}
int ian_encode_pre_vjp_host(ian_handle* h, const float* x, int n, const float* dz_iaf, float* dx) {
  return call_encode_pre_vjp(h, true, x, n, dz_iaf, dx, nullptr);
}
int ian_encode_pre_jvp_dev(ian_handle* h, const float* x, const float* v, int n, float* z_iaf, float* dz_iaf, void* stream) {
  return call_encode_pre_jvp(h, false, x, v, n, z_iaf, dz_iaf, stream);
}
int ian_encode_pre_jvp_host(ian_handle* h, const float* x, const float* v, int n, float* z_iaf, float* dz_iaf) {
  return call_encode_pre_jvp(h, true, x, v, n, z_iaf, dz_iaf, nullptr);
}

// ---- fused all-gather of decoded images over NVLink peer memory ---------------------------------------------
static size_t gather_bytes(int world, int n_local) { return (size_t)2 * world * n_local * 12288 * sizeof(float) + 256; }

int ian_gather_create(ian_handle* h, int world, int rank, int n_local, void* ipc_handle_out) {
  if (!h || !ipc_handle_out) return fail(h, IAN_ERR_INVALID, "NULL argument");
  if (!h->finalized) return fail(h, IAN_ERR_STATE, "ian_finalize() has not been called");
  if (h->model_kind != IAN_MODEL_SIMPLE) return fail(h, IAN_ERR_UNSUPPORTED, "the fused gather is wired into the IAN_simple dec_out kernel");
  if (world < 1 || world > 8 || rank < 0 || rank >= world || n_local < 1 || n_local > 65536)
    return fail(h, IAN_ERR_INVALID, "bad world/rank/n_local (%d,%d,%d)", world, rank, n_local);
  if (h->gbuf) return fail(h, IAN_ERR_STATE, "gather buffers already created");
  DeviceGuard dg(h->device);
  CUDA_TRY(h, cudaMalloc((void**)&h->gbuf, gather_bytes(world, n_local)));
  CUDA_TRY(h, cudaMemset(h->gbuf, 0, gather_bytes(world, n_local)));
  cudaIpcMemHandle_t ipc;
  CUDA_TRY(h, cudaIpcGetMemHandle(&ipc, h->gbuf));
  memcpy(ipc_handle_out, &ipc, sizeof(ipc));
  h->gw = world; h->grank = rank; h->gn = n_local;
  return IAN_OK;
}

int ian_gather_connect(ian_handle* h, const void* all_handles) {
  if (!h || !all_handles || !h->gbuf) return fail(h, IAN_ERR_STATE, "ian_gather_create() first");
  DeviceGuard dg(h->device);
  for (int r = 0; r < h->gw; ++r) {
    if (r == h->grank) { h->gpeer_buf[r] = h->gbuf; continue; }
    cudaIpcMemHandle_t ipc;
    memcpy(&ipc, (const char*)all_handles + (size_t)r * sizeof(ipc), sizeof(ipc));
    void* p = nullptr;
    CUDA_TRY(h, cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess));
    h->gpeer_buf[r] = (float*)p;
  }
  h->gconnected = true;
  return IAN_OK;
}

namespace {
struct GatherSlots { float* dsts[8]; float* flags[8]; size_t half, mine; };
GatherSlots gather_slots(const ian_handle* h) {
  GatherSlots g;
  g.half = (size_t)h->gw * h->gn * 12288;                         // floats per gather buffer
  g.mine = (size_t)h->grank * h->gn * 12288;
  for (int r = 0; r < h->gw; ++r) {
    g.dsts[r] = h->gpeer_buf[r] + (size_t)h->gcur * g.half + g.mine;   // my shard's slot in rank r's current buffer
    g.flags[r] = h->gpeer_buf[r] + 2 * g.half;                    // rank r's flag block (64 ints) after its buffers
  }
  return g;
}

int check_gather_ready(ian_handle* h, const float* x, int n_local) {
  int rc = check_ready(h, n_local, x, x);
  if (rc != IAN_OK) return rc;
  if (!h->gconnected) return fail(h, IAN_ERR_STATE, "ian_gather_connect() has not been called");
  if (n_local != h->gn) return fail(h, IAN_ERR_INVALID, "n_local %d differs from the %d the gather buffers were sized for", n_local, h->gn);
  if (h->path != IAN_PATH_TC) return fail(h, IAN_ERR_UNSUPPORTED, "fused gather runs on the tensor-core path");
  return IAN_OK;
}

// encode -> decode of the local shard (in <= 512-image chunks), dec_out storing into `ndst` destination bases
int run_shard_into(ian_handle* h, const float* x, int n_local, float* z_out, float* const* bases, int ndst, cudaStream_t st) {
  return for_chunks(h, n_local, [&](Plan* pl, int off, int) {
    float* dsts[8];
    for (int r = 0; r < ndst; ++r) dsts[r] = bases[r] + (size_t)off * 12288;
    int rc = run_encode(h, pl, x + (size_t)off * 12288, nullptr, z_out ? z_out + (size_t)off * 100 : pl->z, st);
    if (rc != IAN_OK) return rc;
    h->gather_dsts = dsts; h->gather_ndst = ndst;
    rc = run_decode_from_planes(h, pl, nullptr, st);
    h->gather_dsts = nullptr; h->gather_ndst = 0;
    return rc;
  });
}
}  // namespace

int ian_reconstruct_gather_dev(ian_handle* h, const float* x, int n_local, float* z_out, float** gathered_out, void* stream) {
  if (!gathered_out) return fail(h, IAN_ERR_INVALID, "gathered_out is NULL");
  int rc = check_gather_ready(h, x, n_local);
  if (rc != IAN_OK) return rc;
  DeviceGuard dg(h->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  if (h->g_done_valid[h->gcur]) {                                  // an earlier pipelined step still owns this half
    CUDA_TRY(h, cudaStreamWaitEvent(st, h->g_done[h->gcur], 0));
    h->g_done_valid[h->gcur] = false;
  }
  GatherSlots g = gather_slots(h);
  if ((rc = run_shard_into(h, x, n_local, z_out, g.dsts, h->gw, st)) != IAN_OK) return rc;   // peer stores from dec_out
  h->gepoch += 1;
  LAUNCH_TRY(h, launch_peer_barrier(g.flags, h->gw, h->grank, h->gepoch, st));
  *gathered_out = h->gbuf + (size_t)h->gcur * g.half;
  h->gcur ^= 1;
  h->g_last = -1;
  return IAN_OK;
}

// Pipelined form: the shard is decoded into this rank's own buffer on `stream`; a small copy kernel on a side stream
// then pushes it to every peer while the caller's NEXT step computes.  ian_gather_wait_dev makes `stream` wait for the
// most recent step's gather and returns its buffer.
int ian_reconstruct_gather_async_dev(ian_handle* h, const float* x, int n_local, float* z_out, void* stream) {
  int rc = check_gather_ready(h, x, n_local);
  if (rc != IAN_OK) return rc;
  DeviceGuard dg(h->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  if (!h->push_stream) {
    CUDA_TRY(h, cudaStreamCreateWithFlags(&h->push_stream, cudaStreamNonBlocking));
    for (int b = 0; b < 2; ++b) {
      CUDA_TRY(h, cudaEventCreateWithFlags(&h->g_comp[b], cudaEventDisableTiming));
      CUDA_TRY(h, cudaEventCreateWithFlags(&h->g_done[b], cudaEventDisableTiming));
    }
    if (const char* c = getenv("IAN_PUSH_CTAS")) { int v = atoi(c); if (v >= 1 && v <= tc_num_sms()) h->push_ctas = v; }
    if (const char* c = getenv("IAN_PUSH")) h->push_mode = !strcmp(c, "kernel") ? 1 : 0;
  }
  const int half_id = h->gcur;
  if (h->g_done_valid[half_id]) CUDA_TRY(h, cudaStreamWaitEvent(st, h->g_done[half_id], 0));   // push of step t-2 has read this half
  GatherSlots g = gather_slots(h);
  float* local[1] = {g.dsts[h->grank]};
  if ((rc = run_shard_into(h, x, n_local, z_out, local, 1, st)) != IAN_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->g_comp[half_id], st));
  CUDA_TRY(h, cudaStreamWaitEvent(h->push_stream, h->g_comp[half_id], 0));
  h->gepoch += 1;
  const MemOps& mo = memops();
  if (h->push_mode == 0 && mo.write && mo.wait) {
    // copy engines + stream memory operations: nothing of the push occupies an SM, so the next step's persistent tensor
    // kernels keep all SMs (a co-resident copy KERNEL held its SMs' shared-memory configuration and cost the first three
    // tap-GEMMs of the next step +60 % at 8 GPUs).  Order on the side stream: publish free[t] to every peer; per peer wait
    // for ITS free[t], then DMA the shard into its buffer; publish pushed[t]; wait for everybody's pushed[t].
    CUstream ps = (CUstream)h->push_stream;
    const size_t bytes = (size_t)n_local * 12288 * sizeof(float);
    auto flag = [&](int r, int idx) { return (CUdeviceptr)(uintptr_t)(reinterpret_cast<int*>(g.flags[r]) + idx); };
    for (int k = 1; k < h->gw; ++k) {
      const int p = (h->grank + k) % h->gw;
      if (mo.write(ps, flag(p, 8 + h->grank), (cuuint32_t)h->gepoch, CU_STREAM_WRITE_VALUE_DEFAULT) != CUDA_SUCCESS)
        return fail(h, IAN_ERR_CUDA, "cuStreamWriteValue32(free) failed");
    }
    for (int k = 1; k < h->gw; ++k) {
      const int p = (h->grank + k) % h->gw;
      if (mo.wait(ps, flag(h->grank, 8 + p), (cuuint32_t)h->gepoch, CU_STREAM_WAIT_VALUE_GEQ) != CUDA_SUCCESS)
        return fail(h, IAN_ERR_CUDA, "cuStreamWaitValue32(free) failed");
      CUDA_TRY(h, cudaMemcpyAsync(g.dsts[p], g.dsts[h->grank], bytes, cudaMemcpyDeviceToDevice, h->push_stream));
    }
    for (int p = 0; p < h->gw; ++p)
      if (mo.write(ps, flag(p, 16 + h->grank), (cuuint32_t)h->gepoch, CU_STREAM_WRITE_VALUE_DEFAULT) != CUDA_SUCCESS)
        return fail(h, IAN_ERR_CUDA, "cuStreamWriteValue32(pushed) failed");
    for (int p = 0; p < h->gw; ++p)
      if (mo.wait(ps, flag(h->grank, 16 + p), (cuuint32_t)h->gepoch, CU_STREAM_WAIT_VALUE_GEQ) != CUDA_SUCCESS)
        return fail(h, IAN_ERR_CUDA, "cuStreamWaitValue32(pushed) failed");
  } else {
    LAUNCH_TRY(h, launch_peer_push(g.dsts[h->grank], g.dsts, g.flags, (long long)n_local * 12288, h->gw, h->grank, h->gepoch,
                                   h->push_ctas, h->push_stream));
  }
  CUDA_TRY(h, cudaEventRecord(h->g_done[half_id], h->push_stream));
  h->g_done_valid[half_id] = true;
  h->g_last = half_id;
  h->gcur ^= 1;
  return IAN_OK;
}

int ian_gather_wait_dev(ian_handle* h, float** gathered_out, void* stream) {
  if (!h || !gathered_out) return fail(h, IAN_ERR_INVALID, "NULL argument");
  if (h->g_last < 0) return fail(h, IAN_ERR_STATE, "no pipelined gather step is outstanding");
  DeviceGuard dg(h->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  CUDA_TRY(h, cudaStreamWaitEvent(st, h->g_done[h->g_last], 0));
  *gathered_out = h->gbuf + (size_t)h->g_last * ((size_t)h->gw * h->gn * 12288);
  return IAN_OK;
}

// ---- training-mode pieces (SURVEY 8f rank 4; the trainers themselves stay the reference's) ------------------------------

int ian_bn_batch_stats_dev(ian_handle* h, const float* x, int n, int c, int hw, double* sum, double* sumsq, void* stream) {
  if (!h) return IAN_ERR_INVALID;
  if (!x || !sum || !sumsq || n < 1 || c < 1 || hw < 1) return fail(h, IAN_ERR_INVALID, "bad argument (n=%d c=%d hw=%d)", n, c, hw);
  DeviceGuard dg(h->device);
  int rc = ensure_train_ws(h, bn_workspace_bytes(c));
  if (rc != IAN_OK) return rc;
  LAUNCH_TRY(h, launch_bn_batch_stats(x, n, c, hw, sum, sumsq, h->train_ws, stream ? (cudaStream_t)stream : h->stream));
  return IAN_OK;
}

int ian_bn_train_normalize_dev(ian_handle* h, const float* x, int n, int c, int hw, const double* sum, const double* sumsq,
                               double count, const float* gamma, const float* beta, float eps, float alpha, float* running_mean,
                               float* running_inv_std, float* y, void* stream) {
  if (!h) return IAN_ERR_INVALID;
  if (!x || !y || !sum || !sumsq || n < 1 || c < 1 || hw < 1 || !(count >= 1.0))
    return fail(h, IAN_ERR_INVALID, "bad argument (n=%d c=%d hw=%d count=%g)", n, c, hw, count);
  DeviceGuard dg(h->device);
  int rc = ensure_train_ws(h, bn_workspace_bytes(c));
  if (rc != IAN_OK) return rc;
  LAUNCH_TRY(h, launch_bn_train_normalize(x, n, c, hw, sum, sumsq, count, gamma, beta, eps, alpha, running_mean, running_inv_std, y,
                                          h->train_ws, stream ? (cudaStream_t)stream : h->stream));
  return IAN_OK;
}

int ian_minibatch_discrim_dev(ian_handle* h, const float* x, int n, int d, const float* theta, const float* log_weight_scale,
                              const float* b, int num_kernels, int dim_per_kernel, float* out, void* stream) {
  if (!h) return IAN_ERR_INVALID;
  if (!x || !theta || !log_weight_scale || !b || !out || n < 1 || d < 1 || num_kernels < 1 || dim_per_kernel < 1)
    return fail(h, IAN_ERR_INVALID, "bad argument");
  DeviceGuard dg(h->device);
  int rc = ensure_train_ws(h, mb_workspace_bytes(n, num_kernels, dim_per_kernel));
  if (rc != IAN_OK) return rc;
  LAUNCH_TRY(h, launch_minibatch_discrim(x, n, d, theta, log_weight_scale, b, num_kernels, dim_per_kernel, out, h->train_ws,
                                         stream ? (cudaStream_t)stream : h->stream));
  return IAN_OK;
}

int ian_bn_backward_sums_dev(ian_handle* h, const float* x, const float* dy, int n, int c, int hw, const double* sum, const double* sumsq,
                             double count, float eps, double* sum_dy, double* sum_dyx, float* dgamma, float* dbeta, void* stream) {
  if (!h) return IAN_ERR_INVALID;
  if (!x || !dy || !sum || !sumsq || !sum_dy || !sum_dyx || n < 0 || c < 1 || hw < 1 || !(count >= 1.0))
    return fail(h, IAN_ERR_INVALID, "bad argument (n=%d c=%d hw=%d count=%g)", n, c, hw, count);
  if (n == 0) return IAN_OK;
  DeviceGuard dg(h->device);
  int rc = ensure_train_ws(h, bn_workspace_bytes(c));
  if (rc != IAN_OK) return rc;
  LAUNCH_TRY(h, launch_bn_backward_sums(x, dy, n, c, hw, sum, sumsq, count, eps, sum_dy, sum_dyx, dgamma, dbeta, h->train_ws,
                                        stream ? (cudaStream_t)stream : h->stream));
  return IAN_OK;
}

int ian_bn_backward_dx_dev(ian_handle* h, const float* x, const float* dy, int n, int c, int hw, const double* sum, const double* sumsq,
                           double count, const double* sum_dy, const double* sum_dyx, const float* gamma, float eps, float* dx,
                           void* stream) {
  if (!h) return IAN_ERR_INVALID;
  if (!x || !dy || !dx || !sum || !sumsq || !sum_dy || !sum_dyx || n < 0 || c < 1 || hw < 1 || !(count >= 1.0))
    return fail(h, IAN_ERR_INVALID, "bad argument (n=%d c=%d hw=%d count=%g)", n, c, hw, count);
  if (n == 0) return IAN_OK;
  DeviceGuard dg(h->device);
  int rc = ensure_train_ws(h, bn_workspace_bytes(c));
  if (rc != IAN_OK) return rc;
  LAUNCH_TRY(h, launch_bn_backward_dx(x, dy, n, c, hw, sum, sumsq, count, sum_dy, sum_dyx, gamma, eps, dx, h->train_ws,
                                      stream ? (cudaStream_t)stream : h->stream));
  return IAN_OK;
}

int ian_minibatch_discrim_bwd_dev(ian_handle* h, const float* x, int n, int d, const float* theta, const float* log_weight_scale,
                                  const float* b, int num_kernels, int dim_per_kernel, const float* g, float* dx, float* dtheta,
                                  float* dlog_weight_scale, float* db, void* stream) {
  if (!h) return IAN_ERR_INVALID;
  if (!x || !theta || !log_weight_scale || !b || !g || n < 0 || d < 1 || num_kernels < 1 || dim_per_kernel < 1)
    return fail(h, IAN_ERR_INVALID, "bad argument");
  if (n == 0) return IAN_OK;
  DeviceGuard dg(h->device);
  int rc = ensure_train_ws(h, mb_bwd_workspace_bytes(n, d, num_kernels, dim_per_kernel));
  if (rc != IAN_OK) return rc;
  LAUNCH_TRY(h, launch_minibatch_discrim_bwd(x, n, d, theta, log_weight_scale, num_kernels, dim_per_kernel, g, dx, dtheta,
                                             dlog_weight_scale, db, h->train_ws, stream ? (cudaStream_t)stream : h->stream));
  return IAN_OK;
}

// ---- one NPE paint stroke in one call (reference NPE.py:192-235, photo mode) ---------------------------------
int ian_paint_stroke_host(ian_handle* h, float* z, const int32_t* box, const float* rgb_frame, float weight,
                          const uint8_t* recon_u8, const float* error, uint8_t* im_u8, uint8_t* display_u8) {
  int rc = check_ready(h, 1, z, rgb_frame);
  if (rc != IAN_OK) return rc;
  if (!box || !recon_u8 || !error || !im_u8) return fail(h, IAN_ERR_INVALID, "NULL argument");
  if ((rc = validate_boxes(h, box, 1)) != IAN_OK) return rc;
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  Plan* pl = nullptr;
  if ((rc = get_plan(h, 1, &pl)) != IAN_OK) return rc;
  // staging buffer of the stroke: error (float32) | recon (u8) | IM (u8) | display (u8 HWC)
  if (!pl->stroke) {
    uint8_t* p = nullptr;
    if ((rc = alloc_buf(h, pl, p, 49152 + 12288 + 12288 + 256 * 256 * 3)) != IAN_OK) return rc;
    pl->stroke = p;
  }
  float* d_error = reinterpret_cast<float*>(pl->stroke);
  uint8_t* d_recon = pl->stroke + 49152;
  uint8_t* d_im = d_recon + 12288;
  uint8_t* d_disp = d_im + 12288;
  CUDA_TRY(h, cudaMemcpyAsync(pl->z, z, 400, cudaMemcpyHostToDevice, st));
  CUDA_TRY(h, cudaMemcpyAsync(pl->boxes, box, 16, cudaMemcpyHostToDevice, st));
  CUDA_TRY(h, cudaMemcpyAsync(pl->target, rgb_frame, 12288 * 4, cudaMemcpyHostToDevice, st));
  CUDA_TRY(h, cudaMemcpyAsync(d_recon, recon_u8, 12288, cudaMemcpyHostToDevice, st));
  CUDA_TRY(h, cudaMemcpyAsync(d_error, error, 12288 * 4, cudaMemcpyHostToDevice, st));
  rc = run_graphed(h, pl, Plan::G_STROKE, float_bits(weight), st, [&] {
    LAUNCH_TRY(h, launch_z_to_planes(pl->z, pl->zp.p, pl->zp.plane, 1, st));
    int q = run_grad_core(h, pl, pl->boxes, pl->target, 1, nullptr, st);                                    // NPE.py:205
    if (q != IAN_OK) return q;
    LAUNCH_TRY(h, launch_brush_update(pl->gpad, pl->boxes, weight, nullptr, pl->z, pl->zp.p, pl->zp.plane, 1, st));  // :206-209
    if ((q = run_decode_from_planes(h, pl, pl->xhat, st)) != IAN_OK) return q;                     // NPE.py:218 sample_at
    LAUNCH_TRY(h, launch_npe_blend(pl->xhat, d_recon, d_error, d_im, d_disp, st));                  // NPE.py:218-231
    return (int)IAN_OK;
  });
  if (rc != IAN_OK) return rc;
  CUDA_TRY(h, cudaMemcpyAsync(z, pl->z, 400, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaMemcpyAsync(im_u8, d_im, 12288, cudaMemcpyDeviceToHost, st));
  if (display_u8) CUDA_TRY(h, cudaMemcpyAsync(display_u8, d_disp, 256 * 256 * 3, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaStreamSynchronize(st));
  return IAN_OK;
}

}  // extern "C"
