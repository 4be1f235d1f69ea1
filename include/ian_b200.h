/*
 * ian_b200.h -- C-ABI of libian_b200.so: the H100-native (sm_90a) implementation of the IAN hot path
 * of ajbrock/Neural-Photo-Editor.
 *
 * The reference has NO native boundary for this path: its contract is the Python class API.IAN
 * (reference API.py:11-110), whose methods hand numpy arrays to Theano-compiled functions.  Each entry
 * point below replaces one of those compiled functions; the citation says which.  A host binding
 * (ctypes, cffi, cgo, JNI ...) needs nothing but this header: plain pointers and sizes, int status
 * codes, no C++/torch types.  The Python mirror of API.IAN that ships in this repo
 * (neural-photo-editor_b200/API.py) is such a binding; INTEGRATION.md shows the stub.
 *
 * Conventions
 *   - every function returns IAN_OK (0) or a negative ian_status; ian_last_error() gives the text.
 *   - image tensors are float32 NCHW (n,3,64,64) in [-1,1]; latents are float32 (n,100); row-major.
 *   - *_dev entry points take DEVICE pointers valid on the handle's device and enqueue on `stream`
 *     (a cudaStream_t passed as void*, NULL = the handle's own stream) without synchronising.
 *   - *_host entry points take HOST pointers, do H2D, compute, D2H and return after the result landed
 *     (the numpy-in / numpy-out semantics of the reference's theano.function calls).
 *   - a handle is bound to one device and is not thread-safe (API.IAN is single-threaded: NPE.py calls
 *     it from the Tk main loop).
 *   - results are reproducible: a call repeated with the same batch size returns the same bits (split-K and
 *     stream-K partial sums are added in a fixed order; there are no atomics on the path).
 *   - environment, read by ian_create: IAN_CHUNK=<n> images per internal chunk (default 512); IAN_PATH=simt selects
 *     the FFMA verification kernels; IAN_STREAMK=0 disables stream-K scheduling, IAN_STREAMK=2 uses it on every eligible
 *     launch (tests); IAN_GRAPHS=0 disables the CUDA-graph replay that *_host calls with <= 32 images use;
 *     IAN_SPLITK=0 disables split-K (tests); IAN_PUSH=kernel makes the pipelined all-gather push with a copy kernel
 *     (IAN_PUSH_CTAS=<n> CTAs) instead of copy engines + stream memory operations; IAN_PDL=0 launches the kernel chains
 *     plainly instead of with programmatic dependent launch; IAN_FINALIZE8=0 chooses the one-thread split-K finalize.
 *     All of these select schedules or launch forms of the same kernels (DESIGN.md section 5.8);
 *     results do not depend on IAN_GRAPHS, IAN_PDL or IAN_FINALIZE8 (bit-identical), the others change float32 summation
 *     order within the tolerances of the parity tests.
 *   - stream semantics of *_dev calls: kernels of one call are chained with programmatic dependent launch among themselves;
 *     towards the caller's own work on `stream` (kernels, copies, events before and after the call) the usual stream order
 *     holds -- the first kernel of a call waits for everything enqueued before it before it reads or writes any argument,
 *     and a kernel the caller launches afterwards without the programmatic attribute starts after the call's last kernel
 *     has completed.
 */
#ifndef IAN_B200_H_
#define IAN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ian_handle ian_handle;

typedef enum ian_status {
  IAN_OK = 0,
  IAN_ERR_INVALID = -1,   /* bad argument (shape, NULL, non-integral box, empty box ...)        */
  IAN_ERR_CUDA = -2,      /* CUDA runtime / driver error                                        */
  IAN_ERR_STATE = -3,     /* call order: parameters missing, not finalized ...                  */
  IAN_ERR_UNSUPPORTED = -4
} ian_status;

/* Model graph selector.  Replaces `config_module.get_model(dnn=dnn)` (reference API.py:18-21). */
typedef enum ian_model_kind {
  IAN_MODEL_SIMPLE = 0,   /* reference IAN_simple.py:56-241                                                  */
  IAN_MODEL_FULL = 1,     /* reference IAN.py:67-228: MADE/IAF latent flow, MDC blocks, RGB-Beta head          */
  IAN_MODEL_V1 = 2        /* reference IANv1.py:63-222: MADE/IAF latent flow, plain deconv decoder, RGB-Beta   */
} ian_model_kind;

/* Compute path of the dense contractions (enc_conv2-4, dec_conv1-3, fully-connected layers).
 * Both are CUDA on the GPU; there is no CPU path.
 *   IAN_PATH_TC   : wgmma tensor-core kernels, fp32 emulated by a 3-pass bf16 split (default)
 *   IAN_PATH_SIMT : fp32 FFMA kernels (verification path, bit-for-bit independent of IAN_PATH_TC) */
typedef enum ian_path { IAN_PATH_TC = 0, IAN_PATH_SIMT = 1 } ian_path;

/* ---- lifecycle: replaces IAN.__init__ (reference API.py:12-64) --------------------------------- */

/* Create an empty model on CUDA device `device`. */
int ian_create(int model_kind, int device, ian_handle** out);

/* Upload one parameter under its reference checkpoint name ("enc_conv2.W", "bnorm2.inv_std", ...;
 * names and shapes: reference GANcheckpoints.py:33-57 + IAN_simple.py layer names).  `data` is a HOST
 * float32 array of `ndim` dims `shape`, in the reference's own layout (conv W (Cout,Cin,5,5); deconv W
 * (Cin,Cout,5,5); dense W (in,out)).  Unlike the reference loader (which only warns,
 * GANcheckpoints.py:45-52) a name outside ian_model_param_spec's list or a shape mismatch is an error, and so is a
 * parameter still missing at ian_finalize. */
int ian_set_param(ian_handle* h, const char* name, const float* data, const int64_t* shape, int ndim);

/* The model's OWN parameter list -- what `lasagne.layers.get_all_params(...)` hands GANcheckpoints.load_weights in the
 * reference (API.py:23-30; GANcheckpoints.py:33-57).  A loader iterates index 0..count-1, looks each `name` up in the
 * checkpoint and calls ian_set_param; keys of the file that are not in this list (the trainer's `log_sigma_theta`,
 * discriminator weights, `metadata`) are ignored exactly as the reference loader ignores them.  Handle-free (no GPU
 * needed).  ian_model_param_count returns the count (or a negative ian_status); `name` stays valid for the life of
 * the process; `shape` receives 4 entries (trailing ones are 1). */
int ian_model_param_count(int model_kind);
int ian_model_param_spec(int model_kind, int index, const char** name, int64_t* shape /*[4]*/, int* ndim);

/* IAN_MODEL_FULL / IAN_MODEL_V1: the MADE input ordering (a permutation of 0..99) from which the autoregressive masks are
 * derived by integer comparison (reference mask_generator.py:29-38,93-94).  Replaces the one
 * `shuffle_ordering` draw of `l_IAF_mu/ls.reset("Once")` (reference API.py:33-36).  Must precede ian_finalize. */
int ian_set_made_ordering(ian_handle* h, const int32_t* ordering, int n);

/* The 0/1 autoregressive mask the library derives from `ordering` for one MaskedLayer, as (in,out) bytes [100][100]:
 * which = 0 `<net>_input` (mask_generator.py:93 for layer 0), 1 `<net>_output_W`, 2 `<net>_output_D` (direct
 * input->output, layers.py:822-836).  Pure host integer logic (handle-free): lets a test compare the mask indexing
 * bit for bit with the reference's MaskGenerator. */
int ian_made_mask(const int32_t* ordering, int n, int which, uint8_t* mask_out);
/* Debug getter: the masked MADE weights W*M as uploaded, float32 [2 nets: mu, ls][3: input, output_W, output_D][100][100]. */
int ian_debug_made_weights(ian_handle* h, float* out);

/* Check that every parameter of the graph is present, fold BatchNorm (inference), re-lay weights for
 * the kernels and upload them.  Must precede any compute call. */
int ian_finalize(ian_handle* h);

int ian_destroy(ian_handle* h);
const char* ian_last_error(const ian_handle* h);   /* h may be NULL: last error of ian_create     */

int ian_get_zdim(const ian_handle* h);             /* replaces IAN.get_zdim (API.py:92-96) -> 100 */
int ian_set_path(ian_handle* h, int path);         /* ian_path                                    */
/* Arithmetic of the dense contractions.  IAN_PRECISION_FP32 (default): float32 semantics, every operand kept as
 * bf16 hi|lo planes, 3 tensor-core passes.  IAN_PRECISION_BF16 (full IAN only; BASELINE configs[2]): operands
 * rounded to bf16, one pass, fp32 accumulation -- about 1e-2 max-abs from the float32 result. */
typedef enum ian_precision { IAN_PRECISION_FP32 = 0, IAN_PRECISION_BF16 = 1 } ian_precision;
int ian_set_precision(ian_handle* h, int precision);
/* Number of kernels this library launched on the handle since creation (bench.py gpu_launches). */
int64_t ian_launch_count(const ian_handle* h);

/* ---- encode: replaces Z_hat_fn / IAN.encode_images (reference API.py:50-51, 78-90) ------------- */
/* z = mu(x) (deterministic=True, what API.py:50 compiles).  If eps != NULL the reparameterised
 * sample z = mu + exp(logsigma) * eps (reference layers.py:419-433, eps injected: (n,100)).       */
int ian_encode_dev(ian_handle* h, const float* x, int n, const float* eps, float* z, void* stream);
int ian_encode_host(ian_handle* h, const float* x, int n, const float* eps, float* z);

/* ---- decode: replaces X_hat_fn / IAN.sample_at (reference API.py:46-47, 98-110) ---------------- */
int ian_decode_dev(ian_handle* h, const float* z, int n, float* x, void* stream);
int ian_decode_host(ian_handle* h, const float* z, int n, float* x);

/* ---- encode -> decode in one call (BASELINE metric; no reference equivalent: NPE calls the two
 * functions back to back, NPE.py:257-261) ------------------------------------------------------- */
int ian_reconstruct_dev(ian_handle* h, const float* x, int n, float* z_out /*nullable*/, float* x_hat,
                        void* stream);
int ian_reconstruct_host(ian_handle* h, const float* x, int n, float* z_out /*nullable*/, float* x_hat);

/* ---- pipelined encode -> decode for streaming use (no reference equivalent; the reference is synchronous) --
 * ian_reconstruct_submit enqueues  H2D(x) -> encode -> decode -> D2H(x_hat[, z])  on three streams (copy-in,
 * compute, copy-out) and returns a ticket at once; up to two requests are in flight, so the copies of one request
 * overlap the compute of its neighbours.  ian_reconstruct_wait blocks until that request's outputs have landed in
 * the host buffers, which must stay valid until then.  n <= 512.  Pinned host memory (ian_host_alloc) is what
 * makes the copies asynchronous; pageable memory works but serialises. */
int ian_reconstruct_submit(ian_handle* h, const float* x, int n, float* z_out /*nullable*/, float* x_hat, int* ticket);
int ian_reconstruct_wait(ian_handle* h, int ticket);
/* Page-locked host memory owned by the handle (freed by ian_host_free or ian_destroy). */
int ian_host_alloc(ian_handle* h, size_t bytes, void** out);
int ian_host_free(ian_handle* h, void* p);

/* ---- data-parallel encode -> decode with the all-gather FUSED into the decoder's last kernel (no reference
 * equivalent: the reference is single-GPU).  One process per GPU; every rank calls, in order:
 *   ian_gather_create(h, world, rank, n_local, handle64)   allocate this rank's double gather buffer, get its 64-byte
 *                                                          CUDA IPC handle
 *   (exchange the handles between ranks with any transport, e.g. torch.distributed.all_gather)
 *   ian_gather_connect(h, all_handles)                     map every peer's buffer (NVLink peer access)
 *   ian_reconstruct_gather_dev(h, x, n_local, z, &gathered, stream)   per step
 * The dec_out kernel stores each decoded image straight into slot `rank` of EVERY rank's gather buffer (st.global on
 * peer pointers), then a flag barrier over peer memory makes the step complete: `gathered` (world*n_local,3,64,64)
 * holds all ranks' images on return of the stream work.  n_local may exceed the 512-image plan chunk (the shard then
 * runs as consecutive chunks into the same gather buffer, one barrier at the end).
 * Lifetime of a result: the two gather buffers alternate, so step t+1 of ANY rank never touches the buffer that holds
 * step t -- but a peer that has passed the barrier of step t+1 may begin its step t+2 stores into it.  A result is
 * therefore valid until the stream work of THIS rank's next call has executed: enqueue every consumer of step t on
 * `stream` (or order it before) the call of step t+1.  tests/test_gpu_multi.py skews the ranks to check exactly this. */
int ian_gather_create(ian_handle* h, int world, int rank, int n_local, void* ipc_handle_out /*64 bytes*/);
int ian_gather_connect(ian_handle* h, const void* all_handles /*world x 64 bytes*/);
int ian_reconstruct_gather_dev(ian_handle* h, const float* x, int n_local, float* z_out /*nullable*/, float** gathered_out,
                               void* stream);
/* Pipelined form of the same all-gather, for streams of batches.  dec_out's peer stores are bound by the NVLink
 * egress (7 x 12.6 MB per GPU and step at 8 x 256 images: ~0.11 ms of link time behind a 0.04 ms kernel), so here the
 * shard is decoded into this rank's own buffer and a side stream pushes it to every peer WHILE the next step's tensor
 * kernels run -- by copy engines, with the free/pushed flag handshake that orders the buffer reuse across ranks done as
 * stream memory operations (cuStreamWriteValue32 / cuStreamWaitValue32) on peer-mapped flag words, so that no SM is taken
 * from the persistent tensor kernels (a copy-kernel form exists behind IAN_PUSH=kernel and measured slower for that
 * reason).  ian_reconstruct_gather_async_dev enqueues one step and returns; ian_gather_wait_dev makes `stream`
 * wait until the most recent step's images of ALL ranks have landed and returns that buffer.  A result must be
 * consumed (in stream order) before the call that submits the step after next.  Steps are collective: every rank
 * calls the same sequence of gather entry points. */
int ian_reconstruct_gather_async_dev(ian_handle* h, const float* x, int n_local, float* z_out /*nullable*/, void* stream);
int ian_gather_wait_dev(ian_handle* h, float** gathered_out, void* stream);

/* ---- the function set of the reference's sampling script (reference sample_IAN.py:86-94) ---------------------
 *   Zfn      : X -> l_Z_IAF (deterministic = mu, before the MADE/IAF flow)        -> ian_encode_pre_host
 *   Z_IAF_fn : l_Z_IAF -> l_Z = (z - MADE_mu(z)) / exp(MADE_ls(z))                 -> ian_flow_host(z_out)
 *   sample   : l_Z_IAF -> X (flow, then decoder)                                   -> ian_flow_host(x_out)
 *   sampleZ  : l_Z -> X                                                            -> ian_decode_host
 * For IAN_MODEL_SIMPLE there is no flow: Zfn == encode and Z_IAF_fn is the identity.  The _dev forms run the same kernels
 * as the _host forms (bit-identical results); as for ian_encode_*, n must be positive. */
int ian_encode_pre_dev(ian_handle* h, const float* x, int n, float* z_iaf, void* stream);
int ian_encode_pre_host(ian_handle* h, const float* x, int n, float* z_iaf);
int ian_flow_dev(ian_handle* h, const float* z_iaf, int n, float* z_out /*nullable*/, float* x_out /*nullable*/, void* stream);
int ian_flow_host(ian_handle* h, const float* z_iaf, int n, float* z_out /*nullable*/, float* x_out /*nullable*/);

/* ---- derivatives of the sampling script's functions: the prior space l_Z_IAF --------------------------------------------
 * On IAN.py / IANv1.py the generative prior lives in l_Z_IAF, the input of the MADE/IAF flow (sample_IAN.py feeds N(0,1)
 * noise there and interpolates there).  These split the encoder's derivatives at that boundary:
 *   flow (Z_IAF_fn):   dz_iaf = (d l_Z / d l_Z_IAF)^T . dz          dz = (d l_Z / d l_Z_IAF) . v
 *   Zfn:               dx = (d l_Z_IAF / d x)^T . dz_iaf            dz_iaf = (d l_Z_IAF / d x) . v
 * Zfn is deterministic (l_Z_IAF = mu, no eps).  z_iaf, dz, v (flow), dz_iaf (n,100); x, v (Zfn), dx (n,3,64,64).
 * ian_flow_jvp_*'s z (nullable) receives Z_IAF_fn(z_iaf) and ian_encode_pre_jvp_*'s z_iaf (nullable) Zfn(x), bit for bit.
 * ian_encode_vjp_*(x, dz) equals ian_encode_pre_vjp_*(x, ian_flow_vjp_*(Zfn(x), dz)) and ian_encode_jvp_*(x, v) equals
 * ian_flow_jvp_*(Zfn(x), ian_encode_pre_jvp_*(x, v)) bit for bit, eps absent.  `sample` (l_Z_IAF -> X) has no entry of its
 * own; its derivatives are the compositions
 *   VJP: ian_flow_vjp_*(z_iaf, ian_decode_vjp_*(Z_IAF_fn(z_iaf), dx))      JVP: ian_decode_jvp_*(Z_IAF_fn(z_iaf), ian_flow_jvp_*(z_iaf, v))
 * The flow runs in float32 FFMA in either precision (made_iaf_kernel's summation order, recomputed); its rectify' is 1/2 at
 * exactly 0, as in the encoder VJP and JVP, so ian_flow_vjp_* is the exact transpose of ian_flow_jvp_*'s linear map.  On
 * IAN_MODEL_SIMPLE the flow is the identity: ian_flow_vjp_* returns dz, ian_flow_jvp_* returns v (and z_iaf as z), and the
 * ian_encode_pre_* derivatives return what ian_encode_vjp_* / ian_encode_jvp_* return with eps = NULL.  All three graphs,
 * both paths; bf16 precision on the flow graphs as for ian_encode_vjp_* / ian_encode_jvp_*.  n == 0 does nothing; n < 0 or a
 * NULL required pointer -> IAN_ERR_INVALID; not finalized -> IAN_ERR_STATE.  Deterministic (a repeated call is
 * bit-identical).  The flow entries need no memory beyond a plan's (n,100) buffers; the Zfn entries allocate what
 * ian_encode_vjp_* / ian_encode_jvp_* allocate on their first call per batch size, and share it with them. */
int ian_flow_vjp_dev(ian_handle* h, const float* z_iaf, const float* dz, int n, float* dz_iaf, void* stream);
int ian_flow_vjp_host(ian_handle* h, const float* z_iaf, const float* dz, int n, float* dz_iaf);
int ian_flow_jvp_dev(ian_handle* h, const float* z_iaf, const float* v, int n, float* z /*nullable*/, float* dz, void* stream);
int ian_flow_jvp_host(ian_handle* h, const float* z_iaf, const float* v, int n, float* z /*nullable*/, float* dz);
int ian_encode_pre_vjp_dev(ian_handle* h, const float* x, int n, const float* dz_iaf, float* dx, void* stream);
int ian_encode_pre_vjp_host(ian_handle* h, const float* x, int n, const float* dz_iaf, float* dx);
int ian_encode_pre_jvp_dev(ian_handle* h, const float* x, const float* v, int n, float* z_iaf /*nullable*/, float* dz_iaf,
                           void* stream);
int ian_encode_pre_jvp_host(ian_handle* h, const float* x, const float* v, int n, float* z_iaf /*nullable*/, float* dz_iaf);

/* ---- latent-brush gradients: replace calculate_RGB_gradient / calculate_lighten_gradient
 * (reference API.py:59, 64; IAN.imgrad / IAN.imgradRGB API.py:66-76), batched per sample -------- */
/* boxes: (n,4) int32 rows [c1,r1,c2,r2], half-open box [r1:r2, c1:c2], 0<=c1<c2<=64, 0<=r1<r2<=64.
 * target: NULL -> lighten gradient d/dz mean(x_hat[k,:,box_k]);
 *         target_is_frame=0 -> (n,3) colour per sample, broadcast over the frame;
 *         target_is_frame=1 -> (n,3,64,64) frames (what NPE passes, NPE.py:205).
 * g: (n,100) = d/dz_k mean((target_k[:,box_k] - x_hat[k,:,box_k])^2).                              */
int ian_grad_dev(ian_handle* h, const float* z, const int32_t* boxes, const float* target,
                 int target_is_frame, int n, float* g, void* stream);
int ian_grad_host(ian_handle* h, const float* z, const int32_t* boxes, const float* target,
                  int target_is_frame, int n, float* g);

/* ---- decoder vector-Jacobian product: reverse mode through the decoder from l_Z (reference API.py:46), any cotangent --
 *   dz = (d x_hat / d z)^T . dx_hat
 * z (n,100), dx_hat (n,3,64,64) float32 NCHW, dz (n,100).  The brush gradients above are the special case
 * dx_hat = d loss / d x_hat of a box loss; this takes any pixel-space loss (soft or per-pixel weighted brushes, L1, losses
 * on the whole frame).  Recomputes the forward.  All three graphs, both paths; bf16 precision on the flow graphs as for
 * ian_grad_*.  A box-loss cotangent formed in float32 exactly as the kernels form it (inv = 1/(3*bh*bw); (2*inv)*(x_hat - t)
 * or inv inside the box, 0 outside) gives ian_grad_*'s result bit for bit. */
int ian_decode_vjp_dev(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz, void* stream);
int ian_decode_vjp_host(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz);

/* ---- decoder Jacobian-vector product: forward mode through the decoder from l_Z (reference API.py:46) ----------------
 *   dx_hat = (d x_hat / d z) . v
 * z, v (n,100); dx_hat (n,3,64,64) float32 NCHW; x_hat (n,3,64,64) nullable: receives ian_decode_*(z) bit for bit.  On
 * IAN.py / IANv1.py z is the decoder's input l_Z, as for ian_decode_* and ian_decode_vjp_* (no MADE/IAF).  One batch-100 call
 * with the identity as v gives the 100 columns of the decoder's Jacobian at one latent.  Recomputes the forward; the tangent
 * chain runs the forward's tap-GEMMs on tangent planes.  The derivative conventions are the decoder VJP's (rectify: h > 0;
 * LeakyRectify: the sign of the stored activation, slope 0.2; tanh: 1 - x_hat^2 from the float32 x_hat; the RGB-Beta head's
 * sigmoid and Beta-layer expressions), so <u, JVP(v)> = <ian_decode_vjp_*(u), v> up to float32 summation, also on samples
 * at a rectifier kink.  All three graphs, both paths; bf16 precision on the flow graphs as for ian_decode_vjp_*.
 * n == 0 does nothing; n < 0 or a NULL z, v or dx_hat -> IAN_ERR_INVALID; not finalized -> IAN_ERR_STATE.  Deterministic
 * (a repeated call is bit-identical).  The first call per batch size allocates that plan's tangent planes, maps and
 * split-K slabs: about 1.0 MB per image on IAN_simple, 3.2 MB on IANv1.py and 5.9 MB on IAN.py; plans that never call
 * it keep their memory. */
int ian_decode_jvp_dev(ian_handle* h, const float* z, const float* v, int n, float* x_hat, float* dx_hat, void* stream);
int ian_decode_jvp_host(ian_handle* h, const float* z, const float* v, int n, float* x_hat, float* dx_hat);

/* ---- encoder Jacobian-vector product: forward mode through the encoder (reference API.py:50) ----------------------------
 *   dz = (d z / d x) . v
 * x, v (n,3,64,64) float32 NCHW in the units the graph sees; eps (n,100) nullable; dz (n,100); z (n,100) nullable: receives
 * ian_encode_*(x, eps) bit for bit.  z is what ian_encode_* returns: mu (+ exp(logsigma) eps) on IAN_simple, and the
 * MADE/IAF flow of that on IAN.py / IANv1.py.  eps is a constant input: there is no tangent with respect to it.  Recomputes
 * the forward; the tangent chain runs the forward's tap-GEMMs on tangent planes.  The derivative conventions are the encoder
 * VJP's (LeakyRectify: the sign of the stored activation, slope 0.2; enc_fc1: rectify 1 where f1 > 0 or elu f1 + 1; the
 * flow's rectify 1/2 at exactly 0), so <u, JVP(v)> = <ian_encode_vjp_*(u), v> up to float32 summation.  All three graphs,
 * both paths; bf16 precision on the flow graphs as for ian_encode_vjp_* (enc_conv1 and its tangent stay float32).
 * n == 0 does nothing; n < 0 or a NULL x, v or dz -> IAN_ERR_INVALID; not finalized -> IAN_ERR_STATE.  Deterministic
 * (a repeated call is bit-identical).  The first call per batch size allocates that plan's tangent planes, maps and
 * split-K slabs: the encoder's activations once more, about 1 MB per image (computed from the shapes); plans that never
 * call it keep their memory. */
int ian_encode_jvp_dev(ian_handle* h, const float* x, const float* v, int n, const float* eps, float* z, float* dz, void* stream);
int ian_encode_jvp_host(ian_handle* h, const float* x, const float* v, int n, const float* eps, float* z, float* dz);

/* ---- latent fit: Gauss-Newton normal equations of the decoder and a batched Levenberg-Marquardt fit to images -----------
 * Per sample: z (100) is the decoder's input l_Z, as for ian_decode_* and ian_decode_jvp_* (on IAN.py / IANv1.py after the
 * MADE/IAF flow); x (3,64,64) float32 NCHW is the target in [-1,1]; x_hat = ian_decode_*(z) at the call's batch size,
 * r = x_hat - x (12288 values) and J = d x_hat / d z (12288 x 100), with ian_decode_jvp_*'s derivative conventions.
 *
 * ian_decode_gauss_newton_*: A = J^T J (n,100,100; the decoder's pull-back metric, both triangles), g = J^T r (n,100) and
 *   e = r^T r (n, nullable), float64.  J comes from one batch-100 decoder JVP per sample with the identity as tangents (the
 *   bits of ian_decode_jvp_* on a 100-row batch, what API.IAN.decoder_jacobian returns); A, g and e are float64 sums of
 *   exact float64 products of the float32 J and of r formed in float64, added in a fixed order.
 * ian_fit_latent_*: `iters` Levenberg-Marquardt steps per sample, in place on z (in: the start, out: the fit); loss
 *   (n, iters+1) float32, nullable, receives e / 12288 (the mean squared error) of the start and after every step.  Each
 *   step solves (A + lambda D) delta = -g by a float64 Cholesky factorisation, D = diag(max(A_ii, 1e-9 max_j A_jj)), and
 *   decodes z_trial = float32(z + delta).  If e(z_trial) < e(z) the step is accepted: z <- z_trial, lambda <- max(lambda/10,
 *   1e-7); otherwise (also when a pivot is not positive) z is unchanged and lambda <- min(10 lambda, 1e10).  lambda starts
 *   at 1e-3.  These constants are fixed.  e(z) is the float64 sum of (x_hat - x)^2 in one fixed order, so the loss history
 *   is non-increasing and a step that repeats the previous entry leaves z bit-unchanged.  No host round trip: every
 *   decision is made on the device, per sample.
 * Both: all three graphs, both paths; bf16 precision on the flow graphs as for ian_decode_jvp_* (the normal equations and
 * the solve are float64 in either precision).  n == 0 does nothing; n < 0, iters < 0 or a NULL z, x, A or g ->
 * IAN_ERR_INVALID; not finalized -> IAN_ERR_STATE.  Deterministic (a repeated call is bit-identical; the device form
 * computes the host form's bits).  The first call on a handle allocates 5.0 MB (the identity tangents, J and the Gram's
 * partial sums) and the batch-100 plan with its decoder-JVP tangent planes (what ian_decode_jvp_* allocates at n = 100);
 * the first call per batch size allocates that plan's normal equations and fit state, about 180 KB per image. */
int ian_decode_gauss_newton_dev(ian_handle* h, const float* z, const float* x, int n, double* A, double* g,
                                double* e /*nullable*/, void* stream);
int ian_decode_gauss_newton_host(ian_handle* h, const float* z, const float* x, int n, double* A, double* g,
                                 double* e /*nullable*/);
int ian_fit_latent_dev(ian_handle* h, const float* x, int n, float* z, int iters, float* loss /*nullable*/, void* stream);
int ian_fit_latent_host(ian_handle* h, const float* x, int n, float* z, int iters, float* loss /*nullable*/);

/* ---- masked latent fit under the prior: pixel-weighted Levenberg-Marquardt with a Gaussian prior in the sampling space --
 * Per sample the fit runs in the fit space u (100): l_Z on IAN_simple, l_Z_IAF on IAN.py / IANv1.py (where the sampling
 * script draws N(0, I)), with z = F(u) the MADE/IAF flow of ian_flow_* (the identity on IAN_simple).  With x_hat =
 * decode(F(u)) (the bits of ian_flow_* with x_out at the call's batch size), r = x_hat - x, w (3,64,64) float32 per-pixel
 * weights (NULL: all ones) and prior = beta >= 0 (a double; the pixel-noise variance of a Gaussian likelihood, so the
 * minimiser is the MAP latent under N(0, I)):
 *   E(u) = sum_p w_p r_p^2 + beta |u|^2,   J_u = d x_hat / d u = J_dec(F(u)) J_F(u)   (12288 x 100)
 * Pixels with w_p == 0 contribute exactly nothing: they are skipped, so x may hold anything there, NaN included.
 * ian_map_gauss_newton_*: A = J_u^T W J_u + beta I (n,100,100, both triangles), g = J_u^T W r + beta u (n,100) and e = E(u)
 *   (n, nullable), float64.  J_u comes from one batch-100 pass per sample: u replicated 100 times, the flow's JVP with the
 *   identity as tangents (ian_flow_jvp_*'s kernels), then the decoder JVP with those columns as tangents; on IAN_simple
 *   exactly ian_decode_gauss_newton_*'s pass.  w multiplies one factor of every product (exact in float64), A, g and e are
 *   summed in a fixed order and the prior terms are added once, after the pixel sums.
 * ian_fit_latent_map_*: `iters` Levenberg-Marquardt steps per sample in place on u (in: the start, out: the fit), with
 *   ian_fit_latent_*'s solve, damping, constants and accept / reject rule applied to this A, g and E; trial steps decode
 *   F(u_trial).  z_out (n,100, nullable) receives F(u) of the final u with the bits of ian_flow_* (the l_Z that
 *   ian_decode_*, the brush gradients and the paint stroke take); loss (n, iters+1, nullable) receives E / 12288, prior
 *   term included, of the start and after every step: non-increasing, and a flat entry leaves u bit-unchanged.
 * With w = NULL and prior = 0 on IAN_simple both compute ian_decode_gauss_newton_* / ian_fit_latent_*'s bits; w of all ones
 * computes w = NULL's bits on every graph.
 * Both: all three graphs, both paths; bf16 precision on the flow graphs.  n == 0 does nothing; n < 0, iters < 0, a negative
 * or non-finite prior, or a NULL u, x, A or g -> IAN_ERR_INVALID; the host forms also reject a negative or non-finite
 * weight with IAN_ERR_INVALID (the device forms take w as given); not finalized -> IAN_ERR_STATE.  Deterministic (a
 * repeated call is bit-identical; the device form computes the host form's bits).  Memory: what ian_fit_latent_*
 * allocates, shared with it -- the first call on a handle 5.0 MB and the batch-100 plan with its decoder-JVP tangent planes,
 * plus 80 KB of flow rows on IAN.py / IANv1.py; the first call per batch size about 180 KB per image. */
int ian_map_gauss_newton_dev(ian_handle* h, const float* u, const float* x, const float* w /*nullable*/, double prior, int n,
                             double* A, double* g, double* e /*nullable*/, void* stream);
int ian_map_gauss_newton_host(ian_handle* h, const float* u, const float* x, const float* w /*nullable*/, double prior, int n,
                              double* A, double* g, double* e /*nullable*/);
int ian_fit_latent_map_dev(ian_handle* h, const float* x, const float* w /*nullable*/, double prior, int n, float* u,
                           float* z_out /*nullable*/, int iters, float* loss /*nullable*/, void* stream);
int ian_fit_latent_map_host(ian_handle* h, const float* x, const float* w /*nullable*/, double prior, int n, float* u,
                            float* z_out /*nullable*/, int iters, float* loss /*nullable*/);

/* ---- robust latent fit: Huber and Cauchy pixel losses by reweighted Levenberg-Marquardt ----------------------------------
 * The masked fit above with a robust loss rho on each squared residual, so pixels the generator cannot draw (an occluder, a
 * caption, a highlight) lose their pull on u without anyone marking them.  In the same fit space u, with r, w (NULL: all ones)
 * and prior = beta as there, s = r^2 and a per-sample scale delta:
 *   E(u) = sum_{p: w_p > 0} w_p rho(r_p^2) + beta |u|^2
 *   IAN_ROBUST_HUBER:  rho(s) = s for s <= delta^2, else 2 delta sqrt(s) - delta^2;   rho'(s) = 1, or delta / sqrt(s)
 *   IAN_ROBUST_CAUCHY: rho(s) = delta^2 log1p(s / delta^2);                            rho'(s) = 1 / (1 + s / delta^2)
 * Both rho are concave in s, so with omega_p = w_p rho'(r_p^2) at the current u, sum_p omega_p r_p(u')^2 majorises E up to a
 * constant and Gauss-Newton on it (iteratively reweighted least squares) is sound.
 * scale (n doubles, nullable): delta per sample, > 0 and not NaN; +inf only for Huber, where the loss is exactly the squared
 *   one.  NULL: automatic, taken once at the start and held for the whole fit: delta = max(m c, 1/255) with m the lower median
 *   (rank floor((count - 1) / 2)) of float32 |x_hat - x| over the pixels with w > 0 at the start's x_hat, c = 1.345 * 1.4826
 *   (Huber) or 2.3849 * 1.4826 (Cauchy) -- the 95 %-efficiency constants times the MAD's Gaussian consistency factor -- and
 *   1/255 half an 8-bit level on [-1, 1]; 1/255 when no pixel is weighted (E is then the prior alone).  scale_out (n,
 *   nullable) receives the delta used.
 * ian_robust_gauss_newton_*: A = J_u^T Omega J_u + beta I (n,100,100, both triangles), g = J_u^T Omega r + beta u (n,100)
 *   (= half the gradient of E) and e = E(u) (n, nullable), float64, from ian_map_gauss_newton_*'s J_u pass; omega multiplies
 *   one factor of every product, formed in float64.  With scale NULL delta is automatic at u.
 * ian_fit_latent_robust_*: `iters` Levenberg-Marquardt steps per sample in place on u, with ian_fit_latent_map_*'s solve,
 *   damping, constants and accept / reject rule applied to this A, g and the true E: loss (n, iters+1, nullable) receives
 *   E / 12288 of the start and after every step, non-increasing, and a flat entry leaves u bit-unchanged.  z_out as in
 *   ian_fit_latent_map_*.  outlier_w (n,3,64,64, nullable) receives rho'(r^2) at the final u (1 where the loss is quadratic,
 *   towards 0 on what the latent does not explain) and 0 where w == 0.
 * Huber with every scale +inf computes ian_map_gauss_newton_*'s A and g and ian_fit_latent_map_*'s u, z and loss bits; its e
 * differs from map's by summation order only.  Both: all three graphs, both paths; bf16 precision on the flow graphs.
 * n == 0 does nothing; an unknown kind, n < 0, iters < 0, a negative or non-finite prior, or a NULL u, x, A or g ->
 * IAN_ERR_INVALID; the host forms also check every weight (finite, >= 0) and every scale (the device forms take w and scale as
 * given); not finalized -> IAN_ERR_STATE.  Deterministic (a repeated call is bit-identical; the device form computes the host
 * form's bits); one sample's inputs never change another sample's outputs.  Memory: what ian_fit_latent_map_* allocates,
 * shared with it, plus 8 bytes per image of the plan. */
enum { IAN_ROBUST_HUBER = 1, IAN_ROBUST_CAUCHY = 2 };
int ian_robust_gauss_newton_dev(ian_handle* h, const float* u, const float* x, const float* w /*nullable*/, double prior,
                                int kind, const double* scale /*nullable*/, int n, double* A, double* g, double* e /*nullable*/,
                                double* scale_out /*nullable*/, void* stream);
int ian_robust_gauss_newton_host(ian_handle* h, const float* u, const float* x, const float* w /*nullable*/, double prior,
                                 int kind, const double* scale /*nullable*/, int n, double* A, double* g,
                                 double* e /*nullable*/, double* scale_out /*nullable*/);
int ian_fit_latent_robust_dev(ian_handle* h, const float* x, const float* w /*nullable*/, double prior, int kind,
                              const double* scale /*nullable*/, int n, float* u, float* z_out /*nullable*/, int iters,
                              float* loss /*nullable*/, double* scale_out /*nullable*/, float* outlier_w /*nullable*/,
                              void* stream);
int ian_fit_latent_robust_host(ian_handle* h, const float* x, const float* w /*nullable*/, double prior, int kind,
                               const double* scale /*nullable*/, int n, float* u, float* z_out /*nullable*/, int iters,
                               float* loss /*nullable*/, double* scale_out /*nullable*/, float* outlier_w /*nullable*/);

/* ---- the IAN's introspection features and the latent fit under its feature-wise loss ---------------------------------
 * The features g_1..g_4 are l_introspect = [enc_conv1, enc_conv2, enc_conv3, enc_conv4] of the reference graphs
 * (IAN_simple.py:240, IAN.py:227, IANv1.py:220): the deterministic encoder's activations after BatchNorm (inference
 * statistics, as in Z_hat_fn) and LeakyReLU, with M_i = 131072, 65536, 32768, 16384 elements per image.  Their values are
 * what the encoder stores (float32 mode: exact float32; bf16 mode: the bf16 values the next layer reads).
 * ian_introspect_*: x (n,3,64,64) -> f1 (n,128,32,32), f2 (n,256,16,16), f3 (n,512,8,8), f4 (n,1024,4,4) float32 NCHW, each
 *   nullable: the encoder forward stopped after enc_conv4.
 * ian_introspect_jvp_*: the features (nullable) and their tangents t1..t4 along the image tangents v (n,3,64,64), in the
 *   same layout: ian_encode_jvp_*'s tangent chain stopped after enc_conv4, with its derivative conventions.
 * With z (n,100) the l_Z the decoder takes, x_hat = decode(z), r = x_hat - x, r_i = g_i(x_hat) - g_i(x), a = pixel_weight
 * and b = feature_weight (doubles, finite, >= 0, not both 0):
 *   l_f = (1/4) sum_i |r_i|^2 / M_i   (per sample; train_IAN.py:244 under deterministic=True)
 *   E(z) = a |r|^2 + b 12288 l_f,   J = d x_hat / d z,   J_i = d g_i(x_hat) / d z,   c_i = 3072 b / M_i
 * ian_feature_gauss_newton_*: A = a J^T J + sum_i c_i J_i^T J_i (n,100,100, both triangles), g = a J^T r + sum_i c_i J_i^T r_i
 *   (n,100) and e = E (n, nullable), float64.  Per sample one batch-100 decoder JVP (ian_decode_gauss_newton_*'s pass) and
 *   one batch-100 encoder JVP to enc_conv4 with those 100 rows x_hat as primal and J's columns as tangents; the features of
 *   x and x_hat come from encoder forwards at the call's batch size.  Every product is formed in float64 and summed in a
 *   fixed order.
 * ian_fit_latent_features_*: `iters` Levenberg-Marquardt steps per sample in place on z with ian_fit_latent_*'s solve,
 *   damping, constants and accept / reject rule applied to this A, g and E; loss (n, iters+1, nullable) receives
 *   E / 12288 = a MSE + b l_f of the start and after every step: non-increasing, and a flat entry leaves z bit-unchanged.
 * a = 1, b = 0 computes ian_decode_gauss_newton_* / ian_fit_latent_*'s bits.
 * All four: all three graphs, both paths; bf16 precision on the flow graphs.  n == 0 does nothing; n < 0, iters < 0, a
 * negative or non-finite weight, a = b = 0, or a NULL x, v, t_i, z, A or g -> IAN_ERR_INVALID; not finalized ->
 * IAN_ERR_STATE.  Deterministic (a repeated call is bit-identical; the device form computes the host form's bits).
 * Memory: the host forms of ian_introspect* stage 1.97 MB per image on their first call per batch size; ian_introspect_jvp_*
 * allocates what ian_encode_jvp_* does.  The fit and its normal equations allocate what ian_fit_latent_* does, plus on the
 * first call on a handle 11.2 MB of Gram partials and the batch-100 plan's encoder tangent planes, and on the first call per
 * batch size 1.97 MB per image of stored features. */
int ian_introspect_dev(ian_handle* h, const float* x, int n, float* f1, float* f2, float* f3, float* f4, void* stream);
int ian_introspect_host(ian_handle* h, const float* x, int n, float* f1, float* f2, float* f3, float* f4);
int ian_introspect_jvp_dev(ian_handle* h, const float* x, const float* v, int n, float* f1 /*nullable*/, float* f2 /*nullable*/,
                           float* f3 /*nullable*/, float* f4 /*nullable*/, float* t1, float* t2, float* t3, float* t4,
                           void* stream);
int ian_introspect_jvp_host(ian_handle* h, const float* x, const float* v, int n, float* f1 /*nullable*/, float* f2 /*nullable*/,
                            float* f3 /*nullable*/, float* f4 /*nullable*/, float* t1, float* t2, float* t3, float* t4);
int ian_feature_gauss_newton_dev(ian_handle* h, const float* z, const float* x, int n, double pixel_weight, double feature_weight,
                                 double* A, double* g, double* e /*nullable*/, void* stream);
int ian_feature_gauss_newton_host(ian_handle* h, const float* z, const float* x, int n, double pixel_weight,
                                  double feature_weight, double* A, double* g, double* e /*nullable*/);
int ian_fit_latent_features_dev(ian_handle* h, const float* x, int n, float* z, int iters, double pixel_weight,
                                double feature_weight, float* loss /*nullable*/, void* stream);
int ian_fit_latent_features_host(ian_handle* h, const float* x, int n, float* z, int iters, double pixel_weight,
                                 double feature_weight, float* loss /*nullable*/);

/* ---- vector-Jacobian product of the introspection features --------------------------------------------------------------
 * dx (n,3,64,64) = sum_i (d g_i / d x)^T c_i, with c1..c4 float32 NCHW in ian_introspect_*'s shapes (n,128,32,32),
 * (n,256,16,16), (n,512,8,8), (n,1024,4,4); each nullable (a zero cotangent).  The derivative conventions are
 * ian_introspect_jvp_*'s (LeakyRectify 0.2 from the sign of the stored activation, inference BatchNorm scale), so
 * <c, introspect_jvp(v)> = <introspect_vjp(c), v> up to float32 summation.  The chain is ian_encode_vjp_*'s, entered at the
 * deepest supplied layer L: the encoder forward stops after enc_conv{L}, and each shallower c_i joins the backward chain
 * before that layer's activation derivative.  All four NULL: dx = 0 and nothing else runs.  All three graphs, both paths;
 * bf16 precision on the flow graphs (the cotangents are then rounded to bf16, as the encoder VJP's own gradients are;
 * enc_conv1's adjoint stays float32).  n == 0 does nothing; n < 0 or a NULL x or dx -> IAN_ERR_INVALID; not finalized ->
 * IAN_ERR_STATE.  Deterministic (a repeated call is bit-identical; the device form computes the host form's bits).
 * Memory: the first call per batch size allocates what ian_encode_vjp_* does (shared with it) plus 0.92 MB per image of
 * cotangent planes for layers 1-3; the host form stages its inputs in ian_introspect*_host's 1.97 MB per image. */
int ian_introspect_vjp_dev(ian_handle* h, const float* x, int n, const float* c1 /*nullable*/, const float* c2 /*nullable*/,
                           const float* c3 /*nullable*/, const float* c4 /*nullable*/, float* dx, void* stream);
int ian_introspect_vjp_host(ian_handle* h, const float* x, int n, const float* c1 /*nullable*/, const float* c2 /*nullable*/,
                            const float* c3 /*nullable*/, const float* c4 /*nullable*/, float* dx);

/* ---- the discriminator head l_discrim (IAN_simple.py:225-231, IAN.py:210-216, IANv1.py:203-209) ------------------------
 * ian_set_discriminator_param loads one of the head's four tensors, in the reference's checkpoint names and shapes:
 *   minibatch_discrim.theta (1024,500,5), minibatch_discrim.log_weight_scale (500,5), minibatch_discrim.b (500),
 *   discrimi.W (1524,U) with U = 1 on IAN_simple / IANv1 (sigmoid) and U = 3 on IAN.py (softmax; train_IAN.py:482-484's
 *   classes: column 0 real, 1 reconstruction, 2 generated).
 * Valid before or after ian_finalize; a second call replaces the tensor (after synchronising the device).  A wrong name or
 * shape -> IAN_ERR_INVALID and nothing changes.  The head is not part of ian_model_param_spec's list.
 *
 * ian_discriminate_*: x (n,3,64,64) -> logits (n,U) = [pool(a4) | f] W and p (n,U, nullable) = sigmoid or softmax(logits),
 *   l_discrim under deterministic=True: a4 is enc_conv4 after inference BatchNorm and LeakyReLU (introspect's f4), pool the
 *   mean over its 4 x 4 pixels (GlobalPoolLayer), f (n,500) the MinibatchLayer's features of the pooled batch
 *   (layers.py:486-524, as ian_minibatch_discrim_dev).  The trunk runs chunk by chunk; the MinibatchLayer and the dense
 *   layer run once over the whole call, in float32 (FFMA, fixed summation order, softmax with its max subtracted).
 * ian_discriminate_vjp_*: dx (n,3,64,64) = (d logits / d x)^T dlogits (n,U) over the whole coupled batch: per chunk the
 *   trunk and pool, over the call the dense layer's and the MinibatchLayer's adjoints, per chunk again the trunk's reverse
 *   chain from enc_conv4 (ian_introspect_vjp_*'s with c4 only).  The trunk's forward runs twice: 2 forwards + 1 backward.
 * BATCH COUPLING: unlike every other entry point, one sample's result depends on the other samples of the call, which form
 *   the MinibatchLayer's minibatch whatever the chunk size.  At n == 1, f = b exactly (the self-pair's exp(-1e6) is 0) and
 *   the MinibatchLayer adds nothing to dx.  One non-finite image makes every sample's f, and so every logit, non-finite.  A
 *   cotangent on sample i reaches every image.  The per-sample isolation that holds elsewhere does not apply here.
 * Both graphs' trunks run on both paths; bf16 precision applies to the trunk where the handle allows it, the head always
 *   runs in float32.  No CUDA graphs.  n == 0 does nothing; n < 0 or a NULL x, logits, dlogits or dx -> IAN_ERR_INVALID;
 *   not finalized or no head loaded (all four tensors) -> IAN_ERR_STATE.  Deterministic (a repeated call is bit-identical;
 *   the device form computes the host form's bits).
 * Memory: 16.3 KB per image of whole-call buffers plus 64 KB per image of the largest chunk (grown to the largest n asked
 *   for); the MinibatchLayer's workspace, shared with ian_minibatch_discrim*_dev: 4 (K P (n + 1)) bytes forward and
 *   4 (K P (2n + d + 1) + K n (n-1)/2) bytes in the VJP (K = 500, P = 5, d = 1024): about 80 MB at n = 256 and 1.1 GB at
 *   n = 1024; the VJP allocates what ian_introspect_vjp_* does for c4. */
int ian_set_discriminator_param(ian_handle* h, const char* name, const float* data, const int64_t* shape, int ndim);
int ian_discriminate_dev(ian_handle* h, const float* x, int n, float* logits, float* p /*nullable*/, void* stream);
int ian_discriminate_host(ian_handle* h, const float* x, int n, float* logits, float* p /*nullable*/);
int ian_discriminate_vjp_dev(ian_handle* h, const float* x, int n, const float* dlogits, float* dx, void* stream);
int ian_discriminate_vjp_host(ian_handle* h, const float* x, int n, const float* dlogits, float* dx);

/* ---- the discriminator in training mode: l_discrim under deterministic=False (train_IAN.py:139-149, train_IAN_simple.py:405)
 * ian_discriminate_train_*: logits and p (nullable) as ian_discriminate_*, with bnorm2..4 in the trunk normalising with the
 *   BATCH's statistics: per channel mean and biased variance over (n, h, w) of enc_conv{2,3,4}'s raw output, inv_std =
 *   1/sqrt(var + 1e-4), y = (x - mean) (gamma inv_std) + beta, then LeakyReLU(0.2); enc_conv1, GlobalPool, the MinibatchLayer
 *   and the dense head are unchanged.  The handle's running mean / inv_std are neither used nor changed.
 *   stats (nullable) receives the statistics used, float32 (2,1792): row 0 the means of bnorm2 (256) | bnorm3 (512) |
 *   bnorm4 (1024), row 1 their inv_std -- Lasagne's running-average update (alpha = 0.1) is the caller's to apply.
 * ian_discriminate_train_vjp_*: dx (n,3,64,64) = (d logits / d x)^T dlogits (n,U) over the whole batch, the gradient flowing
 *   through the batch mean and variance as Theano's T.grad gives it.  1 trunk forward + 1 backward.
 * The sums are float64 per image, added in image order: the statistics, and so every result, do not depend on IAN_CHUNK.
 * BATCH COUPLING as for ian_discriminate_*, and more: every BatchNorm of the trunk couples the samples, so even at n == 1
 *   a sample's result is its own batch's (a 1-image batch normalises over its pixels alone).
 * Precision, paths, argument checks, error codes and IAN_ERR_STATE without a head are ian_discriminate_*'s; n == 0 does
 *   nothing.  Deterministic.  No CUDA graphs.
 * Memory: the whole-call buffers of ian_discriminate_* plus 852 KB per image (enc_conv2..4's raw sums, two cotangent
 *   buffers, float32) and 16 KB per image of partial sums: about 220 MB at n = 256; the VJP allocates what
 *   ian_encode_vjp_* does on each chunk's plan. */
int ian_discriminate_train_dev(ian_handle* h, const float* x, int n, float* logits, float* p /*nullable*/,
                               float* stats /*nullable*/, void* stream);
int ian_discriminate_train_host(ian_handle* h, const float* x, int n, float* logits, float* p /*nullable*/,
                                float* stats /*nullable*/);
int ian_discriminate_train_vjp_dev(ian_handle* h, const float* x, int n, const float* dlogits, float* dx, void* stream);
int ian_discriminate_train_vjp_host(ian_handle* h, const float* x, int n, const float* dlogits, float* dx);

/* ---- decoder parameter vector-Jacobian product (IAN_MODEL_SIMPLE): dL/dtheta for the decoder's trainable tensors -----
 * The parameters train_IAN_simple.py:353 hands to the optimiser (`decoder_params`): l_dec_fc2.W, dec_conv1..3.W, dec_out.W
 * and bnorm_dec_fc2 / bnorm_dc1..3 .beta / .gamma, on the deterministic graph of X_hat_fn (API.py:46): inference
 * BatchNorm, mean / inv_std constant.  z (n,100), dx_hat (n,3,64,64) float32 NCHW as for ian_decode_vjp_*; dz (n,100)
 * nullable, bit for bit ian_decode_vjp_*'s.  grads is indexed like ian_model_param_spec (ian_model_param_count entries,
 * NULL = not wanted; grads itself may be NULL); grads[i] receives parameter i in the reference layout and shape.  A
 * non-NULL entry for a parameter without a gradient -> IAN_ERR_INVALID; IAN_MODEL_FULL / IAN_MODEL_V1 ->
 * IAN_ERR_UNSUPPORTED; n == 0 does nothing.  Results are overwritten, not accumulated (a batch above the plan chunk is summed
 * chunk by chunk in chunk order).  Both paths; deterministic (a repeated call is bit-identical).  The first call per batch
 * size allocates the gradient buffers of that plan (about 2 MB per image plus split-K slabs of at most 64 MB); the first
 * host call also allocates 75 MB of device gradients on the handle, the first call of either 136 KB of BatchNorm statistics. */
/* 1 if ian_decode_param_vjp_* computes a gradient for parameter `index` of ian_model_param_spec (handle-free). */
int ian_param_vjp_supported(int model_kind, int index);
int ian_decode_param_vjp_dev(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz, float* const* grads,
                             void* stream);
int ian_decode_param_vjp_host(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz, float* const* grads);
/* Replace one IAN_simple decoder parameter of a FINALIZED handle: the 13 above or bnorm_dec_fc2 / bnorm_dc1..3 .mean /
 * .inv_std, in the reference layout and shape.  Re-derives what ian_finalize derives from it and writes it into the same
 * device buffers, so plans and captured graphs stay valid; afterwards every entry point computes bit for bit what a handle
 * finalized from the updated parameters computes.  Synchronises the device first (ordered after all earlier work).
 * Other names -> IAN_ERR_INVALID; not finalized -> IAN_ERR_STATE; IAN_MODEL_FULL / IAN_MODEL_V1 -> IAN_ERR_UNSUPPORTED. */
int ian_update_param_host(ian_handle* h, const char* name, const float* data, const int64_t* shape, int ndim);

/* ---- the IAN_simple decoder in training mode: get_output(l_out, {l_Z: z}) under deterministic=False, as the reference's
 * trainers build X_hat and the generated samples (train_IAN_simple.py:217-224, 253) ------------------------------------
 * ian_decode_train_*: x_hat (n,3,64,64) float32 NCHW for z (n,100), with bnorm_dec_fc2 and bnorm_dc1..3 normalising with
 *   the BATCH's statistics: bnorm_dec_fc2 each of its 16384 features over the n samples, bnorm_dc1..3 each channel over
 *   (n, h, w); biased variance, inv_std = 1/sqrt(var + 1e-4), y = (x - mean) (gamma inv_std) + beta, then rectify.
 *   The handle's running mean / inv_std are neither used nor changed.
 *   stats (nullable) receives the statistics used, float32 (2,17280): row 0 the means of bnorm_dec_fc2 (16384, in the
 *   reference's feature order) | bnorm_dc1 (512) | bnorm_dc2 (256) | bnorm_dc3 (128), row 1 their inv_std.  Lasagne's
 *   running-average update, r <- 0.9 r + 0.1 batch for both mean and inv_std, is the caller's to apply
 *   (ian_update_param_host).
 * ian_decode_train_vjp_*: dz (n,100, nullable) = (d x_hat / d z)^T dx_hat through the batch statistics, and the gradients
 *   of ian_decode_param_vjp_*'s 13 tensors on this graph: grads indexed and laid out as there, with its error rules (a
 *   pointer for a parameter without a gradient -> IAN_ERR_INVALID).  Weight gradients run only for the tensors asked for.
 *   1 forward + 1 backward.
 * The sums are float64 per image, added in image order: the statistics, x_hat and dz do not depend on IAN_CHUNK; the
 * weight gradients add the chunks in chunk order.
 * BATCH COUPLING: one sample's z changes every sample's x_hat, and one non-finite z makes every output non-finite.  At
 *   n == 1 bnorm_dec_fc2 sees a single sample, so x_hat = h(beta) does not depend on z: dz and l_dec_fc2.W's gradient are
 *   exactly 0.
 * IAN_MODEL_FULL / IAN_MODEL_V1 -> IAN_ERR_UNSUPPORTED; n == 0 does nothing.  Float32 on both paths.  Deterministic.  No
 *   CUDA graphs.
 * Memory: whole-call buffers of 1.9 MB per image (the four layers' raw sums, 245 760 floats; two cotangent slots the
 *   layers alternate between, 131 072 floats for bnorm_dc3 / bnorm_dc1 and 65 536 for bnorm_dc2 / bnorm_dec_fc2; 256 KB of
 *   float64 partial sums) plus 1.3 MB fixed, grown to the largest batch asked for; the VJP also allocates
 *   ian_decode_param_vjp_*'s buffers on each chunk's plan. */
int ian_decode_train_dev(ian_handle* h, const float* z, int n, float* x_hat, float* stats /*nullable*/, void* stream);
int ian_decode_train_host(ian_handle* h, const float* z, int n, float* x_hat, float* stats /*nullable*/);
int ian_decode_train_vjp_dev(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz /*nullable*/,
                             float* const* grads /*nullable*/, void* stream);
int ian_decode_train_vjp_host(ian_handle* h, const float* z, const float* dx_hat, int n, float* dz /*nullable*/,
                              float* const* grads /*nullable*/);

/* ---- encoder vector-Jacobian product: reverse mode through the encoder from the image (reference Z_hat, API.py:50) ------
 *   dx = (d z / d x)^T . dz
 * x (n,3,64,64) float32 NCHW, eps (n,100) nullable, dz (n,100), dx (n,3,64,64).  z is exactly what ian_encode_* returns for
 * the same x and eps: mu (+ exp(logsigma) * eps) on IAN_simple; on IAN.py / IANv1.py the MADE/IAF flow of that.  No
 * gradient w.r.t. eps.  Recomputes the forward.  All three graphs, both paths; bf16 precision on the flow graphs as for
 * ian_grad_* (enc_conv1 and its adjoint always run in float32).  The first call on a handle builds the backward weight
 * tiles from the forward ones on the device; the first call per batch size allocates its gradient buffers (~1 MB/image). */
int ian_encode_vjp_dev(ian_handle* h, const float* x, int n, const float* eps, const float* dz, float* dx, void* stream);
int ian_encode_vjp_host(ian_handle* h, const float* x, int n, const float* eps, const float* dz, float* dx);

/* ---- latent edit loop: n_steps of the NPE paint rule (reference NPE.py:199-209) per sample:
 *        g = grad(z);  z <- z - weight * g * (1 + (c2 - c1))        (all float32)
 * in place on z (n,100).  `weight` = 0.05 in NPE.py:199.                                          */
int ian_edit_loop_dev(ian_handle* h, float* z, const int32_t* boxes, const float* target,
                      int target_is_frame, int n, int n_steps, float weight, void* stream);
int ian_edit_loop_host(ian_handle* h, float* z, const int32_t* boxes, const float* target,
                       int target_is_frame, int n, int n_steps, float weight);

/* ---- one NPE paint stroke in ONE call: replaces the body of paint() in photo mode (reference NPE.py:199-231):
 *   g = imgradRGB(box, rgb_frame, z);  z <- z - weight * g * (1 + (c2 - c1));  x_hat = sample_at(z)
 *   DELTA = x_hat - to_tanh(RECON);  MASK = gaussian_filter(min(mean_c|DELTA|, 1), 0.7)
 *   IM = uint8(from_tanh(to_tanh(RECON) + MASK*DELTA + (1-MASK)*ERROR))
 * z (1,100) in/out; box int32[4] = [c1,r1,c2,r2]; rgb_frame (1,3,64,64) float32 in [-1,1]; recon_u8 (3,64,64) uint8;
 * error (3,64,64) float32; im_u8 (3,64,64) uint8 out; display_u8 (256,256,3) uint8 out (nullable): IM upsampled 4x
 * nearest-neighbour in HWC order, what update_photo() hands to PIL (NPE.py:107-118).  IAN_MODEL_SIMPLE only. */
int ian_paint_stroke_host(ian_handle* h, float* z, const int32_t* box, const float* rgb_frame, float weight,
                          const uint8_t* recon_u8, const float* error, uint8_t* im_u8, uint8_t* display_u8);

/* ---- training-mode pieces (no trainer here: train_IAN*.py stay the reference's; these are the two forward ops whose
 * training form differs from the deterministic graphs everything above runs).  Device pointers, float32.
 *
 * BatchNorm with BATCH statistics = lasagne BatchNormLayer.get_output_for(deterministic=False), i.e. every BN(...) of
 * reference IAN_simple.py:84-170 / layers.py:411-416 in training.  x is (n, c, hw) (NCHW with hw = H*W; dense layers: hw = 1).
 *   ian_bn_batch_stats_dev      per-channel sum and sum of squares (float64 [c] each) over (n, hw), accumulated in float64
 *                               from the first term (every partial, per thread included): warp-shuffle reductions, fixed
 *                               order, bit-reproducible.  Data-parallel ranks all-reduce the two arrays here
 *                               (cross-GPU synchronised BN) and pass the GLOBAL element count to the second call.
 *   ian_bn_train_normalize_dev  mean = sum/count, inv_std = 1/sqrt(sumsq/count - mean^2 + eps)  (biased variance);
 *                               y = (x - mean) * (gamma * inv_std) + beta;  running_mean / running_inv_std (nullable) are
 *                               updated in place: r <- (1 - alpha) r + alpha * batch value.  lasagne: eps 1e-4, alpha 0.1.
 *                               Accuracy: the variance's float64 cancellation, relative ~1e-16 (|mean|/std)^2; then the
 *                               float32 roundings of mean, gamma * inv_std and x - mean, which the reference also performs.
 *                               A constant channel gives y = beta exactly.
 * The three calls share one workspace per handle, so, like every other entry point, a handle serves one stream at a time.
 * ian_minibatch_discrim_dev     MinibatchLayer.get_output_for(init=False) of reference layers.py:486-524:
 *                               x (n,d), theta (d,K,P), log_weight_scale (K,P), b (K) -> out (n, d+K) = [x | f]. */
int ian_bn_batch_stats_dev(ian_handle* h, const float* x, int n, int c, int hw, double* sum, double* sumsq, void* stream);
int ian_bn_train_normalize_dev(ian_handle* h, const float* x, int n, int c, int hw, const double* sum, const double* sumsq,
                               double count, const float* gamma /*nullable*/, const float* beta /*nullable*/, float eps,
                               float alpha, float* running_mean /*nullable*/, float* running_inv_std /*nullable*/, float* y,
                               void* stream);
int ian_minibatch_discrim_dev(ian_handle* h, const float* x, int n, int d, const float* theta, const float* log_weight_scale,
                              const float* b, int num_kernels, int dim_per_kernel, float* out, void* stream);

/* ---- reverse mode of the two training-mode ops (DESIGN §5.6b).  Same conventions as the forward calls: device pointers,
 * float32 tensors, float64 sums, the handle's workspace and stream; bit-reproducible; what the forward rejects ->
 * IAN_ERR_INVALID; n == 0 does nothing.  Gradients flow through the batch mean and variance (Theano's T.grad through
 * lasagne's input.mean / input.var); the running-average update has none.
 *   ian_bn_backward_sums_dev    this rank's per-channel Σdy and Σdy·x (float64 [c] each) over (n, hw): exact products,
 *                               float64 from the first term, the forward's split order.  sum / sumsq / count / eps are the
 *                               forward's (global after an all-reduce).  dgamma = Σ dy·x̂ = s (Σdy·x - mean Σdy), evaluated in
 *                               float64, and dbeta = Σdy (nullable, float32 [c]) are this rank's: DDP reduces them itself.
 *                               Data-parallel ranks all-reduce sum_dy / sum_dyx here.
 *   ian_bn_backward_dx_dev      from the (global) backward sums, N = count, s = 1/sqrt(var + eps), x̂ = (x - mean) s:
 *                               dx = gamma s (dy - Σdy/N - x̂ Σ(dy x̂)/N), per element in float64, one rounding.
 *                               gamma NULL means 1 (its gradient is then not wanted either).
 * ian_minibatch_discrim_bwd_dev g = dL/d[x | f] (n, d+K) -> dx (n,d), dtheta (d,K,P), dlog_weight_scale (K,P), db (K), each
 *                               nullable.  Recomputes A = x W; each pair i < j forms e_ijk = exp(-Σ_p|A_ikp - A_jkp|) once;
 *                               dA_ikp = -Σ_{j≠i} (g_f[i,k] + g_f[j,k]) e_ijk sgn(A_ikp - A_jkp) with sgn(0) = 0; dx = g_x + dA Wᵀ,
 *                               dW = xᵀ dA, then through W = theta exp(lws) / |theta[:,k,p]|.  FFMA, fixed-order chunked sums,
 *                               no atomics.  b is the forward's (no gradient depends on it).  Workspace: 4 (K P (2n + d) +
 *                               K n (n-1)/2) bytes. */
int ian_bn_backward_sums_dev(ian_handle* h, const float* x, const float* dy, int n, int c, int hw, const double* sum, const double* sumsq,
                             double count, float eps, double* sum_dy, double* sum_dyx, float* dgamma /*nullable*/,
                             float* dbeta /*nullable*/, void* stream);
int ian_bn_backward_dx_dev(ian_handle* h, const float* x, const float* dy, int n, int c, int hw, const double* sum, const double* sumsq,
                           double count, const double* sum_dy, const double* sum_dyx, const float* gamma /*nullable*/, float eps,
                           float* dx, void* stream);
int ian_minibatch_discrim_bwd_dev(ian_handle* h, const float* x, int n, int d, const float* theta, const float* log_weight_scale,
                                  const float* b, int num_kernels, int dim_per_kernel, const float* g, float* dx /*nullable*/,
                                  float* dtheta /*nullable*/, float* dlog_weight_scale /*nullable*/, float* db /*nullable*/,
                                  void* stream);

/* ---- measurement helpers ----------------------------------------------------------------------- */
/* Average device time (ms, CUDA events on the launch stream) of the tap-GEMM kernel of layer
 * `layer_name` ("enc_conv2", "dec_conv1", ...; the encoder VJP's "bwd_enc_head", "bwd_enc_fc1", "bwd_enc_conv4",
 * "bwd_enc_conv3", "bwd_enc_conv2"; "enc_conv1", "dec_out", "brush_seed" -- the loss-seed kernel of the brush gradients
 * and of ian_decode_vjp_* -- "enc_conv1_bwd" -- enc_conv1's adjoint in ian_encode_vjp_* -- for the edge kernels; "wgrad_l_dec_fc2", "wgrad_dec_conv1",
 * "wgrad_dec_conv2", "wgrad_dec_conv3" and "wgrad_dec_out" for the weight gradients of ian_decode_param_vjp_*; in
 * ian_decode_jvp_* "jvp_<layer>" for the tangent tap-GEMM of each decoder forward layer -- "jvp_l_dec_fc2", "jvp_dec_conv1",
 * "jvp_full_dec_conv1", "jvp_dec_conv2a2", ... -- plus "dec_out_jvp" (IAN_simple) and "rgb_head_jvp" (the head's three
 * convolutions on the tangent of its feature map, IAN.py / IANv1.py); in ian_encode_jvp_* "jvp_enc_conv1" (enc_conv1's
 * tangent) and "jvp_enc_conv2", "jvp_enc_conv3", "jvp_enc_conv4", "jvp_enc_fc1", "jvp_enc_head"; in the latent fit "gn_gram"
 * (the normal equations' Gram of one sample, with its chunk reduction) and "gn_solve" (the Levenberg-Marquardt solve of
 * the batch); in the masked fit "map_gram" (the weighted Gram of one sample, with its reduction and the prior terms) and
 * "gn_solve"; in the feature fit "feat_gram" (the feature layers' Gram of one sample, with its reduction and the pixel
 * Gram's weighting), "feat_accept" (the trial objective and accept rule of the batch), "gn_gram" and "gn_solve"; in
 * ian_introspect_vjp_* "feat_cotangent" (the cotangents' conversion to split planes), "introspect_bwd_enc_conv4",
 * "introspect_bwd_enc_conv3", "introspect_bwd_enc_conv2" (a backward GEMM joined by a supplied cotangent; one without
 * runs as "bwd_enc_conv*"), "enc_conv1" and "enc_conv1_bwd"; in the robust fit "robust_gram" (the reweighted Gram of
 * one sample, with its reduction and the prior terms), "robust_scale" (the automatic scale of the batch) and "gn_solve"; in
 * ian_discriminate_* "disc_pool" (a4's pool, per chunk), "disc_mb" (the MinibatchLayer), "disc_head" (the dense layer and
 * its nonlinearity), and in ian_discriminate_vjp_* also "disc_head_bwd", "disc_mb_bwd" and "disc_cotangent" (enc_conv4's
 * cotangent, per chunk) next to the trunk's own layers; in ian_discriminate_train* "disc_train_enc_conv2..4" (the
 * layers' raw sums), "disc_train_stats", "disc_train_norm" (BatchNorm + LeakyReLU into the next layer's planes), and in the
 * VJP also "disc_train_cotangent", "disc_train_bn_bwd" (Σdy, Σdy·x), "disc_train_bn_dx", "disc_train_bwd_enc_conv4..3"; in
 * ian_decode_train* "dec_train_l_dec_fc2", "dec_train_dec_conv1..3" (the layers' raw sums), "dec_train_stats",
 * "dec_train_norm" (BatchNorm + rectify into the next layer's planes) and "dec_out", and in the VJP also "brush_seed",
 * "dec_train_cotangent" (bnorm_dc3's dy), "dec_train_bn_bwd" (Σdy, Σdy·x), "dec_train_bn_grads" (d beta, d gamma),
 * "dec_train_bn_dx", "dec_train_bwd_dec_conv3..1" and the "wgrad_*" of ian_decode_param_vjp_*) over the launches since the last reset; returns <0 if the layer was never timed.  Timing is enabled with ian_set_layer_timing(h, 1). */
int ian_set_layer_timing(ian_handle* h, int enable);
double ian_layer_time_ms(ian_handle* h, const char* layer_name, int reset);

#ifdef __cplusplus
}
#endif
#endif /* IAN_B200_H_ */
