// cfgpp_b200 — C ABI of the AutoencoderKL decoder (include/cfgpp_b200.h, "AutoencoderKL decoder").
#include "capi_util.h"
#include "vae.cuh"

using namespace cfgpp;

struct cfgpp_vae_handle {
  VaeDecoder vae;
  cfgpp_vae_handle(const cfgpp_vae_desc& d, int device) : vae(d, device) {}
};

extern "C" {

CFGPP_API int cfgpp_vae_create(const cfgpp_vae_desc* desc, int device, cfgpp_vae_handle** out) {
  return guarded([&] {
    CFGPP_REQUIRE(desc && out, "null argument");
    *out = new cfgpp_vae_handle(*desc, device);
  });
}

CFGPP_API int cfgpp_vae_destroy(cfgpp_vae_handle* h) {
  return guarded([&] { delete h; });
}

CFGPP_API int cfgpp_vae_load_weight(cfgpp_vae_handle* h, const char* key, const void* data, const int64_t* shape,
                                    int ndim, int dtype, void* stream) {
  return guarded([&] { h->vae.load_weight(key, data, shape, ndim, dtype, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_vae_finalize_weights(cfgpp_vae_handle* h, void* stream) {
  return guarded([&] { h->vae.finalize_weights((cudaStream_t)stream); });
}

CFGPP_API int cfgpp_vae_decode(cfgpp_vae_handle* h, const void* z, int z_dtype, int batch, int h_lat, int w_lat,
                               void* image, void* stream) {
  return guarded([&] { h->vae.decode(z, z_dtype, batch, h_lat, w_lat, (__half*)image, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_vae_encode(cfgpp_vae_handle* h, const void* image, int image_dtype, int batch, int height, int width,
                               const void* noise, void* latent, void* stream) {
  return guarded([&] {
    h->vae.encode(image, image_dtype, batch, height, width, (const __half*)noise, (float*)latent, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_vae_stats(cfgpp_vae_handle* h, double* flops, size_t* workspace_bytes) {
  return guarded([&] {
    if (flops) *flops = h->vae.flops();
    if (workspace_bytes) *workspace_bytes = h->vae.workspace_bytes();
  });
}

// ---- operator-level entry points (one kernel launch each, on the caller's stream) ----
CFGPP_API int cfgpp_op_vae_latent_prep(const void* z, int z_dtype, float scaling, const void* w, const void* bias,
                                       void* out, int B, int HW, void* stream) {
  return guarded([&] {
    run_vae_latent_prep(z, z_dtype == CFGPP_F16 ? 1 : 0, scaling, (const __half*)w, (const __half*)bias, (__half*)out,
                        B, HW, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_vae_row_softmax(void* s, int rows, int n, float scale, void* stream) {
  return guarded([&] {
    run_vae_row_softmax((__half*)s, rows, n, scale * 1.4426950408889634f, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_vae_conv_rgb(const void* x, const void* w, const void* bias, void* out, int B, int H, int W, int C,
                                    void* stream) {
  return guarded([&] {
    run_vae_conv_rgb((const __half*)x, (const __half*)w, (const __half*)bias, (__half*)out, B, H, W, C,
                     (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_vae_image_pad(const void* x, int x_dtype, void* out, int B, int H, int W, void* stream) {
  return guarded([&] { run_vae_image_pad(x, x_dtype == CFGPP_F16 ? 1 : 0, (__half*)out, B, H, W, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_op_vae_moments_sample(const void* x, const void* w, const void* bias, const void* wq, const void* bq,
                                          const void* noise, float scaling, float* out, int B, int H, int W, int C,
                                          void* stream) {
  return guarded([&] {
    run_vae_moments_sample((const __half*)x, (const __half*)w, (const __half*)bias, (const __half*)wq,
                           (const __half*)bq, (const __half*)noise, scaling, out, B, H, W, C, (cudaStream_t)stream);
  });
}

}  // extern "C"
