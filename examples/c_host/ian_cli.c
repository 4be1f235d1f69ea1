/* A host program in plain C over the C-ABI of libian_b200.so -- no Python, no torch: the shape a maintainer's own
 * binding (cgo / JNI / N-API ...) takes.  It mirrors what the reference's API.IAN does around its compiled Theano
 * functions (reference API.py:23-47 load the weights, :50-54 encode / sample_at):
 *
 *   ian_cli <weights.bin> <images.f32> <n> <x_hat.f32> [z.f32]
 *
 * weights.bin : u32 count, then per array: u32 name_len, name, u32 ndim, i64 shape[ndim], f32 data (C order) --
 *               the arrays of the reference's IAN_simple.npz (tests/test_gpu_c_host.py writes it).
 * images.f32  : n x 3 x 64 x 64 float32 in [-1, 1]   (what API.IAN.encode_images receives)
 * x_hat.f32   : the reconstructions, z.f32 : the latents (n x 100).
 * `ian_cli --symbols` only resolves every entry point of include/ian_b200.h (link check; needs no GPU).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "ian_b200.h"

static int die(const char* what, ian_handle* h) {
  const char* e = ian_last_error(h);
  fprintf(stderr, "ian_cli: %s: %s\n", what, e ? e : "?");
  if (h) ian_destroy(h);
  return 1;
}

static float* read_f32(const char* path, size_t count) {
  FILE* f = fopen(path, "rb");
  float* p;
  if (!f) return NULL;
  p = (float*)malloc(count * sizeof(float));
  if (p && fread(p, sizeof(float), count, f) != count) { free(p); p = NULL; }
  fclose(f);
  return p;
}

static int load_weights(ian_handle* h, const char* path) {
  FILE* f = fopen(path, "rb");
  unsigned count, k;
  if (!f) { fprintf(stderr, "ian_cli: cannot open %s\n", path); return -1; }
  if (fread(&count, 4, 1, f) != 1) { fclose(f); return -1; }
  for (k = 0; k < count; ++k) {
    unsigned name_len, ndim, d;
    char name[256];
    int64_t shape[8];
    size_t elems = 1;
    float* data;
    int rc;
    if (fread(&name_len, 4, 1, f) != 1 || name_len >= sizeof(name) || fread(name, 1, name_len, f) != name_len) break;
    name[name_len] = 0;
    if (fread(&ndim, 4, 1, f) != 1 || ndim > 8 || fread(shape, 8, ndim, f) != ndim) break;
    for (d = 0; d < ndim; ++d) elems *= (size_t)shape[d];
    data = (float*)malloc(elems * sizeof(float));
    if (!data || fread(data, sizeof(float), elems, f) != elems) { free(data); break; }
    rc = ian_set_param(h, name, data, shape, (int)ndim);
    free(data);
    if (rc != IAN_OK) { fclose(f); return rc; }
  }
  fclose(f);
  if (k != count) { fprintf(stderr, "ian_cli: %s is truncated or malformed (array %u of %u)\n", path, k, count); return -1; }
  return IAN_OK;
}

/* every entry point of the header, taken by address: an entry point missing from the library fails the link */
typedef void (*anyfn)(void);
static int symbols(void) {
  anyfn fn[] = {
      (anyfn)ian_create, (anyfn)ian_set_param, (anyfn)ian_set_made_ordering, (anyfn)ian_finalize,
      (anyfn)ian_destroy, (anyfn)ian_last_error, (anyfn)ian_get_zdim, (anyfn)ian_set_path,
      (anyfn)ian_set_precision, (anyfn)ian_launch_count, (anyfn)ian_encode_dev,
      (anyfn)ian_encode_host, (anyfn)ian_decode_dev, (anyfn)ian_decode_host,
      (anyfn)ian_reconstruct_dev, (anyfn)ian_reconstruct_host, (anyfn)ian_reconstruct_submit,
      (anyfn)ian_reconstruct_wait, (anyfn)ian_host_alloc, (anyfn)ian_host_free,
      (anyfn)ian_gather_create, (anyfn)ian_gather_connect, (anyfn)ian_reconstruct_gather_dev,
      (anyfn)ian_encode_pre_host, (anyfn)ian_flow_host, (anyfn)ian_grad_dev, (anyfn)ian_grad_host,
      (anyfn)ian_edit_loop_dev, (anyfn)ian_edit_loop_host, (anyfn)ian_paint_stroke_host,
      (anyfn)ian_set_layer_timing, (anyfn)ian_layer_time_ms, (anyfn)ian_model_param_count,
      (anyfn)ian_model_param_spec, (anyfn)ian_made_mask, (anyfn)ian_debug_made_weights,
      (anyfn)ian_reconstruct_gather_async_dev, (anyfn)ian_gather_wait_dev, (anyfn)ian_bn_batch_stats_dev,
      (anyfn)ian_bn_train_normalize_dev, (anyfn)ian_minibatch_discrim_dev, (anyfn)ian_decode_vjp_dev,
      (anyfn)ian_decode_vjp_host, (anyfn)ian_encode_vjp_dev, (anyfn)ian_encode_vjp_host,
      (anyfn)ian_param_vjp_supported, (anyfn)ian_decode_param_vjp_dev, (anyfn)ian_decode_param_vjp_host, (anyfn)ian_update_param_host,
      (anyfn)ian_decode_jvp_dev, (anyfn)ian_decode_jvp_host, (anyfn)ian_encode_jvp_dev, (anyfn)ian_encode_jvp_host,
      (anyfn)ian_encode_pre_dev, (anyfn)ian_flow_dev, (anyfn)ian_flow_vjp_dev, (anyfn)ian_flow_vjp_host, (anyfn)ian_flow_jvp_dev,
      (anyfn)ian_flow_jvp_host, (anyfn)ian_encode_pre_vjp_dev, (anyfn)ian_encode_pre_vjp_host, (anyfn)ian_encode_pre_jvp_dev,
      (anyfn)ian_encode_pre_jvp_host, (anyfn)ian_decode_gauss_newton_dev, (anyfn)ian_decode_gauss_newton_host,
      (anyfn)ian_fit_latent_dev, (anyfn)ian_fit_latent_host, (anyfn)ian_map_gauss_newton_dev, (anyfn)ian_map_gauss_newton_host,
      (anyfn)ian_fit_latent_map_dev, (anyfn)ian_fit_latent_map_host, (anyfn)ian_introspect_dev, (anyfn)ian_introspect_host,
      (anyfn)ian_introspect_jvp_dev, (anyfn)ian_introspect_jvp_host, (anyfn)ian_feature_gauss_newton_dev,
      (anyfn)ian_feature_gauss_newton_host, (anyfn)ian_fit_latent_features_dev, (anyfn)ian_fit_latent_features_host,
      (anyfn)ian_introspect_vjp_dev, (anyfn)ian_introspect_vjp_host, (anyfn)ian_robust_gauss_newton_dev,
      (anyfn)ian_robust_gauss_newton_host, (anyfn)ian_fit_latent_robust_dev, (anyfn)ian_fit_latent_robust_host,
      (anyfn)ian_bn_backward_sums_dev, (anyfn)ian_bn_backward_dx_dev, (anyfn)ian_minibatch_discrim_bwd_dev,
      (anyfn)ian_set_discriminator_param, (anyfn)ian_discriminate_dev, (anyfn)ian_discriminate_host,
      (anyfn)ian_discriminate_vjp_dev, (anyfn)ian_discriminate_vjp_host, (anyfn)ian_discriminate_train_dev,
      (anyfn)ian_discriminate_train_host, (anyfn)ian_discriminate_train_vjp_dev, (anyfn)ian_discriminate_train_vjp_host,
      (anyfn)ian_decode_train_dev, (anyfn)ian_decode_train_host, (anyfn)ian_decode_train_vjp_dev,
      (anyfn)ian_decode_train_vjp_host};
  size_t i, n = sizeof(fn) / sizeof(fn[0]);
  for (i = 0; i < n; ++i)
    if (!fn[i]) return 1;
  printf("%u entry points resolved\n", (unsigned)n);
  return 0;
}

int main(int argc, char** argv) {
  ian_handle* h = NULL;
  float *x, *xh, *z;
  int n, zdim = 0;
  FILE* f;
  if (argc == 2 && !strcmp(argv[1], "--symbols")) return symbols();
  if (argc < 5) {
    fprintf(stderr, "usage: %s <weights.bin> <images.f32> <n> <x_hat.f32> [z.f32]\n       %s --symbols\n", argv[0], argv[0]);
    return 2;
  }
  n = atoi(argv[3]);
  if (n <= 0) { fprintf(stderr, "ian_cli: n must be positive\n"); return 2; }
  if (ian_create(IAN_MODEL_SIMPLE, 0, &h) != IAN_OK) return die("ian_create", NULL);   /* no GPU: fails loudly, no fallback */
  if (load_weights(h, argv[1]) != IAN_OK) return die("loading weights", h);
  if (ian_finalize(h) != IAN_OK) return die("ian_finalize", h);
  zdim = ian_get_zdim(h);
  if (zdim <= 0) return die("ian_get_zdim", h);
  x = read_f32(argv[2], (size_t)n * 12288);
  xh = (float*)malloc((size_t)n * 12288 * sizeof(float));
  z = (float*)malloc((size_t)n * (size_t)zdim * sizeof(float));
  if (!x || !xh || !z) { fprintf(stderr, "ian_cli: cannot read %d images from %s\n", n, argv[2]); ian_destroy(h); return 1; }
  if (ian_reconstruct_host(h, x, n, z, xh) != IAN_OK) return die("ian_reconstruct_host", h);
  f = fopen(argv[4], "wb");
  if (!f || fwrite(xh, sizeof(float), (size_t)n * 12288, f) != (size_t)n * 12288) { fprintf(stderr, "ian_cli: cannot write %s\n", argv[4]); return 1; }
  fclose(f);
  if (argc > 5) {
    f = fopen(argv[5], "wb");
    if (!f || fwrite(z, sizeof(float), (size_t)n * (size_t)zdim, f) != (size_t)n * (size_t)zdim) { fprintf(stderr, "ian_cli: cannot write %s\n", argv[5]); return 1; }
    fclose(f);
  }
  printf("reconstructed %d image(s), zdim %d, %lld kernel launches\n", n, zdim, (long long)ian_launch_count(h));
  free(x); free(xh); free(z);
  ian_destroy(h);
  return 0;
}
