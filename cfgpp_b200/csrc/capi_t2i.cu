// cfgpp_b200 — C ABI of the T2I-Adapter (include/cfgpp_b200.h, "T2I-Adapter") and its kernels' operator-level entries.
#include "capi_util.h"
#include "t2i_adapter.cuh"

using namespace cfgpp;

struct cfgpp_t2i_adapter_handle {
  T2IAdapter adapter;
  cfgpp_t2i_adapter_handle(const cfgpp_t2i_adapter_desc& d, int device) : adapter(d, device) {}
};

extern "C" {

CFGPP_API int cfgpp_t2i_adapter_create(const cfgpp_t2i_adapter_desc* desc, int device, cfgpp_t2i_adapter_handle** out) {
  return guarded([&] {
    CFGPP_REQUIRE(desc && out, "null argument");
    *out = new cfgpp_t2i_adapter_handle(*desc, device);
  });
}

CFGPP_API int cfgpp_t2i_adapter_destroy(cfgpp_t2i_adapter_handle* ad) {
  return guarded([&] { delete ad; });
}

CFGPP_API int cfgpp_t2i_adapter_load_weight(cfgpp_t2i_adapter_handle* ad, const char* key, const void* data,
                                            const int64_t* shape, int ndim, int dtype, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(ad && key && data && shape, "null argument");
    ad->adapter.load_weight(key, data, shape, ndim, dtype, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_t2i_adapter_finalize_weights(cfgpp_t2i_adapter_handle* ad, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(ad != nullptr, "null handle");
    ad->adapter.finalize_weights((cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_t2i_adapter_forward(cfgpp_t2i_adapter_handle* ad, const void* image, int dtype, int batch, int H,
                                        int W, float scale, void* const* features_out, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(ad != nullptr, "null handle");
    ad->adapter.forward(image, dtype, batch, H, W, scale, reinterpret_cast<__half* const*>(features_out),
                        (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_t2i_adapter_stats(cfgpp_t2i_adapter_handle* ad, double* flops, size_t* workspace_bytes) {
  return guarded([&] {
    CFGPP_REQUIRE(ad != nullptr, "null handle");
    if (flops) *flops = ad->adapter.flops();
    if (workspace_bytes) *workspace_bytes = ad->adapter.workspace_bytes();
  });
}

// ---- operator-level entry points (one kernel launch each, on the caller's stream) ----
CFGPP_API int cfgpp_op_pixel_unshuffle(const void* x, int dtype, void* out, int B, int C, int H, int W, int f,
                                       void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "fp16 or fp32 input");
    run_pixel_unshuffle(x, dtype == CFGPP_F16 ? 1 : 0, (__half*)out, B, C, H, W, f, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_avgpool2x2(const void* x, void* out, int B, int H, int W, int C, void* stream) {
  return guarded([&] { run_avgpool2x2((const __half*)x, (__half*)out, B, H, W, C, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_op_relu(void* x, size_t n, void* stream) {
  return guarded([&] { run_relu((__half*)x, n, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_op_scale(const void* x, float s, void* out, size_t n, void* stream) {
  return guarded([&] { run_scale((const __half*)x, s, (__half*)out, n, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_op_t2i_add(void* h, const void* feat, int NB, int B, size_t per_image, const int* on,
                               void* stream) {
  return guarded([&] { run_t2i_add((__half*)h, (const __half*)feat, NB, B, per_image, on, (cudaStream_t)stream); });
}

}  // extern "C"
