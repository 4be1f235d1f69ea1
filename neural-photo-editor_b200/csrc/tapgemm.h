// tapgemm.h -- the "shifted-tap GEMM": the one dense contraction every heavy IAN layer reduces to.
//
//   out[n, p*osh+oh0, q*osw+ow0, co] = epi( sum_t sum_c A[n, (p+dh_t)*sh + vh_t, (q+dw_t)*sw + vw_t, c]
//                                                   * B[wtile_t][co][c] )
//
// with zero padding outside A.  It covers (reference file:line of the op each case replaces):
//   * 5x5 stride-2 convolution, enc_conv2-4 (IAN_simple.py:84-116): 25 taps over the 4 stride-2
//     "views" of the input (view = parity of the input row/col), one phase;
//   * 5x5 stride-2 transposed convolution, dec_conv1-3 (layers.py:436-483): 4 output sub-pixel phases
//     with 9/6/6/4 taps each over the plain input, output written at stride 2;
//   * its backward-data for the latent brush (T.grad at API.py:59,64): a stride-2 5x5 conv again;
//   * dense layers enc_fc1 / enc_mu|logsigma / l_dec_fc2 / dz (IAN_simple.py:117-135): 1 tap, 1x1 grid.
//
// Operands are bf16 SPLIT PLANES: a float32 value v is stored as hi=bf16(v), lo=bf16(v-hi) in two
// planes of the same NHWC tensor (4 bytes/element, 16 significand bits).  The tensor-core path
// computes hi*hi + lo*hi + hi*lo with fp32 accumulation (3 wgmma per K step); the SIMT path
// computes (hi+lo)*(hi+lo) in fp32 FFMA.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

namespace ian {

enum Act : int { ACT_NONE = 0, ACT_LRELU = 1, ACT_RELU = 2, ACT_ELU = 3, ACT_MASK = 4 };

// Function attributes (max dynamic shared memory) and the SM count are PER DEVICE, and one process may hold handles on
// several GPUs (API.IAN(..., device=k)): every launcher keeps its one-time setup in an array indexed by the current
// device.  Setting an attribute twice is harmless, so the flags only need to be tear-free.
constexpr int kMaxDevices = 64;
inline int cur_device() {
  int d = 0;
  cudaGetDevice(&d);
  return (d >= 0 && d < kMaxDevices) ? d : 0;
}
struct DeviceOnce {
  std::atomic<bool> done[kMaxDevices];
  bool is_done(int dev) const { return done[dev].load(std::memory_order_acquire); }
  void set_done(int dev) { done[dev].store(true, std::memory_order_release); }
};

// Programmatic dependent launch (PDL).  A step is a chain of 13-15 short kernels on one stream; with plain launches each
// boundary costs the launch latency plus the next kernel's prologue (barrier init, first descriptor
// fetch) plus the previous kernel's tail, with the SMs idle.  Kernels on the hot chains therefore
//   * call pdl_trigger() first thing (griddepcontrol.launch_dependents: "my successor may be scheduled as soon as every
//     CTA of mine has said so or exited" -- for the persistent kernels that means: as my CTAs retire, SM by SM), and
//   * call pdl_wait() (griddepcontrol.wait: the predecessor grid has COMPLETED and its memory is visible) after their own
//     prologue and before the first global access that is not a constant weight.  Completion is transitive (a grid cannot
//     complete before its own wait returned), so one wait orders a kernel after everything earlier on the stream; it also
//     covers write-after-read on shared scratch (split-K / stream-K workspaces).
// and are launched through launch_pdl(), which sets cudaLaunchAttributeProgrammaticStreamSerialization when the calling
// thread's pdl_flag() is on (the handle turns it off while capturing graphs or timing layers).  A kernel launched
// WITHOUT the attribute is a full stream dependency as ever, and both instructions are no-ops in it: every kernel that is
// not in the list below (flow backward, training pieces, peer barriers, copies, events) still separates the chain.
inline bool& pdl_flag() {
  static thread_local bool on = false;
  return on;
}
// split-K finalize: the cooperative (8 lanes per output) form for deep splits; off = the one-thread form everywhere.  Both
// add the slabs in the same order (tests/test_gpu_parity.py compares them bit for bit); handle-controlled like pdl_flag().
inline bool& coop_finalize_flag() {
  static thread_local bool on = true;
  return on;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_flag() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

constexpr int kMaxTaps = 40;
constexpr int kMaxPhases = 4;

struct Tap {
  int16_t view;   // 0..3 = (row parity << 1) | col parity of the strided input view
  int16_t dh, dw; // shift in view coordinates
  int16_t wtile;  // which [Cout][Cin] weight tile
};

struct Phase {
  int tap_begin, ntaps;
  int oh0, ow0;   // output offset of this phase
};

struct TapGemm {
  // A: NHWC split planes
  const __nv_bfloat16* a;
  long long a_plane;            // elements between hi and lo plane
  int n_img, Hin, Win, Cin;     // Cin % 64 == 0
  int sh, sw;                   // view stride (1 or 2)
  int Hg, Wg;                   // M grid: rows m = (n*Hg + p)*Wg + q
  // B: [wtile][Cout][Cin] split planes, K(=Cin)-major
  const __nv_bfloat16* b;
  long long b_plane;
  int Cout;                     // % 64 == 0 (padded by the host); 16 for the 2-filter RGB-Beta head convs
  int nphase;
  Phase phase[kMaxPhases];
  Tap taps[kMaxTaps];
  // epilogue: v = acc*scale[si] + shift[si]; v = act(v); ACT_MASK: v = acc*scale[si] * (mask>0)
  const float* scale;
  const float* shift;
  int scale_pix_stride;         // si = co + (oh*Wout+ow)*scale_pix_stride
  int act;
  const __nv_bfloat16* mask;    // hi plane with the output's geometry (ACT_MASK): v = acc*scale * (mask > 0 ? 1 : mask_slope)
  float mask_slope;             // 0: rectify backward; 0.2: LeakyRectify(0.2) backward (the mask is the forward ACTIVATION,
                                // whose sign is the pre-activation's)
  int res_after;                // 1: `res` is added AFTER the mask/scale (gradient joining a residual branch) instead of before
                                // BatchNorm (MDBLOCK forward)
  // output: NHWC split planes and/or fp32, pixel = (n*Hout + p*osh+oh0)*Wout + q*osw+ow0
  __nv_bfloat16* out;
  long long out_plane;
  float* out_f32;
  int Hout, Wout, osh, osw;
  // split-K (tensor-core path, small-M layers): K split s stores its raw accumulators to slab s of ws
  // ([ksplit][pixel][Cout], slab stride ws_slab floats); a finalize kernel adds the slabs in split order and
  // applies the epilogue -- no atomics, no zero-fill, bit-reproducible.
  int ksplit;
  float* ws;
  long long ws_slab;
  // MDBLOCK support (reference layers.py:411-416): `res` (output geometry, split planes) is added to the sum
  // before scale/shift; `out_raw` receives the un-normalised sum (the block's residual input x)
  const __nv_bfloat16* res;
  long long res_plane;
  __nv_bfloat16* out_raw;
  long long out_raw_plane;
  // tile-blocked channel-major float32 output [m-tile][cout_real][128 rows] (columns >= cout_real dropped): every
  // 128-row tile owns one contiguous block and a warp writes 128 contiguous bytes per column.  Row order inside a
  // tile and tile order follow tile_shape() below.  Used for the RGB-Beta head's tap table.
  float* out_f32_t;
  int cout_real;
  int out_t_bf16;               // 1: the same table stored as bf16 (single-pass bf16 mode: halves the head's HBM round trip)
  int passes;                   // 3 = float32 via bf16 hi|lo split (default), 1 = plain bf16 (hi planes only)
  // stream-K (see WorkIter in tapgemm_tc.cu): per-CTA partial-sum slots [cta][8][32][BN/2] fp32, arrival flags
  // [cta][8] holding the epoch of the launch that wrote them; sk_ws == nullptr selects whole-tile scheduling
  float* sk_ws;
  int* sk_flags;
  int sk_epoch;
  int sk_force;                 // 1: stream-K on every eligible launch, skipping the makespan test (tests use it)
  // 1: whole tiles of a plain epilogue (scale/shift + none/LReLU/ReLU/ELU into `out` only) leave through TMA stores
  // straight from the accumulators (tensor-core path, float32 mode).  The caller sets the wish (IAN_EPI_TMA=0 clears
  // it); launch_tapgemm_tc keeps it only where the layer qualifies.  Both forms compute the same bits.
  int epi_tma;
};

// 128-row M tiles are boxes {Nt images, Ht rows, Wt cols} of the (n, p, q) output grid
__host__ __device__ inline void tile_shape(int Hg, int Wg, int& Wt, int& Ht, int& Nt) {
  Wt = Wg < 128 ? Wg : 128;
  Ht = Hg < 128 / Wt ? Hg : 128 / Wt;
  Nt = 128 / (Wt * Ht);
}

__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case ACT_LRELU: return 0.6f * v + 0.4f * fabsf(v);       // lasagne LeakyRectify(0.2): f1*x+f2*|x|
    case ACT_RELU:  return 0.5f * (v + fabsf(v));            // lasagne rectify
    case ACT_ELU:   return v > 0.f ? v : expm1f(v);
    default:        return v;
  }
}

__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// ---- launchers (each returns the number of kernels it launched, or <0 on error) -----------------
int launch_tapgemm_simt(const TapGemm& g, cudaStream_t st);
// tensor-core path; maps are built by tc_build_maps() once per plan.  Its K steps run chunk-major: step `it` of a phase
// is channel chunk it / ntaps of tap it % ntaps (split-K and stream-K ranges are cut on that index).
struct TcMaps;   // opaque: CUtensorMaps for A views, B and (where a map can describe it) the output planes
TcMaps* tc_build_maps(const TapGemm& g, char* err, int errlen);
void tc_free_maps(TcMaps*);
int launch_tapgemm_tc(const TapGemm& g, const TcMaps* maps, cudaStream_t st);
int launch_splitk_finalize(const TapGemm& g, cudaStream_t st);
int tc_tile_width(const TcMaps* maps);
int tc_num_sms();
size_t tc_sk_workspace_floats();   // per handle: one 128 x 256 fp32 slot per SM
size_t tc_sk_flag_ints();

// ---- weight gradient of a forward tap-GEMM (wgrad_tc.cu) -------------------------------------------
//   dB[wtile_t][co][ci] = sum_{n,p,q} G[n, p*osh+oh0, q*osw+ow0, co] * A[n, (p+dh_t)*sh+vh_t, (q+dw_t)*sw+vw_t, ci]
// One GEMM per tap: M = Cout, N = Cin, K = the forward M grid (n*Hg*Wg pixels of the tap's phase).  G is dL/d(raw output)
// of the forward layer `f`; its A operand (taps, views, zero padding) is the forward's.  Every weight tile must belong to
// exactly one (phase, tap), so no sum across taps is needed (taps_deconv_s2, taps_dense; wgrad_build_maps checks it).
// K split s writes raw float32 sums to slab s of ws ([ksplit][ntiles][Cout][Cin]); launch_wgrad_finalize adds the slabs in
// split order and scatters into the reference layout -- no atomics, bit-reproducible.
struct WgradGemm {
  TapGemm f;
  const __nv_bfloat16* gr;      // split planes with the forward output's geometry (n, Hout, Wout, Cout)
  long long gr_plane;
  int ksplit;
  float* ws;
  long long ws_slab;            // ntiles * Cout * Cin
};
enum WgradLayout { WG_DECONV = 0,   // dW[ci][co][t] = dB[t][co][ci]  (DeconvLayer W (Cin, Cout, 5, 5))
                   WG_FC2 = 1 };    // l_dec_fc2: dW[k][c*16 + hw] = dB[0][hw*1024 + c][k], k < 100
struct WgradMaps;   // opaque: CUtensorMaps of G (one per phase) and A (one per view)
WgradMaps* wgrad_build_maps(const WgradGemm& w, char* err, int errlen);
void wgrad_free_maps(WgradMaps*);
int wgrad_kboxes(const WgradGemm& w);   // 64-pixel K steps per tap on the tensor-core path
int wgrad_choose_ksplit(const WgradGemm& w, long long max_ws_floats);
int launch_wgrad_tc(const WgradGemm& w, const WgradMaps* maps, cudaStream_t st);
int launch_wgrad_simt(const WgradGemm& w, cudaStream_t st);
int launch_wgrad_finalize(const WgradGemm& w, int layout, float* out, int accumulate, cudaStream_t st);

}  // namespace ian
