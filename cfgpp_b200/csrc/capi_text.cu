// cfgpp_b200 — C ABI of the CLIP text towers (include/cfgpp_b200.h, "CLIP text encoder").
#include "capi_util.h"
#include "text_encoder.cuh"

using namespace cfgpp;

struct cfgpp_clip_handle {
  ClipTextEncoder enc;
  cfgpp_clip_handle(const cfgpp_clip_desc& d, int device) : enc(d, device) {}
};

extern "C" {

CFGPP_API int cfgpp_clip_create(const cfgpp_clip_desc* desc, int device, cfgpp_clip_handle** out) {
  return guarded([&] {
    CFGPP_REQUIRE(desc && out, "null argument");
    *out = new cfgpp_clip_handle(*desc, device);
  });
}

CFGPP_API int cfgpp_clip_destroy(cfgpp_clip_handle* h) {
  return guarded([&] { delete h; });
}

CFGPP_API int cfgpp_clip_load_weight(cfgpp_clip_handle* h, const char* key, const void* data, const int64_t* shape,
                                     int ndim, int dtype, void* stream) {
  return guarded([&] { h->enc.load_weight(key, data, shape, ndim, dtype, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_clip_finalize_weights(cfgpp_clip_handle* h, void* stream) {
  return guarded([&] { h->enc.finalize_weights((cudaStream_t)stream); });
}

CFGPP_API int cfgpp_clip_encode(cfgpp_clip_handle* h, const int32_t* input_ids, const int32_t* pooled_index, int batch,
                                int n_tokens, int skip, void* hidden_out, void* last_hidden_out, void* pooled_out,
                                void* stream) {
  return guarded([&] {
    h->enc.encode(input_ids, pooled_index, batch, n_tokens, skip, (__half*)hidden_out, (__half*)last_hidden_out,
                  (__half*)pooled_out, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_clip_stats(cfgpp_clip_handle* h, double* flops, size_t* workspace_bytes) {
  return guarded([&] {
    if (flops) *flops = h->enc.flops();
    if (workspace_bytes) *workspace_bytes = h->enc.workspace_bytes();
  });
}

struct cfgpp_clip_vision_handle {
  ClipVisionEncoder enc;
  cfgpp_clip_vision_handle(const cfgpp_clip_vision_desc& d, int device) : enc(d, device) {}
};

CFGPP_API int cfgpp_clip_vision_create(const cfgpp_clip_vision_desc* desc, int device, cfgpp_clip_vision_handle** out) {
  return guarded([&] {
    CFGPP_REQUIRE(desc && out, "null argument");
    *out = new cfgpp_clip_vision_handle(*desc, device);
  });
}

CFGPP_API int cfgpp_clip_vision_destroy(cfgpp_clip_vision_handle* h) {
  return guarded([&] { delete h; });
}

CFGPP_API int cfgpp_clip_vision_load_weight(cfgpp_clip_vision_handle* h, const char* key, const void* data,
                                            const int64_t* shape, int ndim, int dtype, void* stream) {
  return guarded([&] { h->enc.load_weight(key, data, shape, ndim, dtype, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_clip_vision_finalize_weights(cfgpp_clip_vision_handle* h, void* stream) {
  return guarded([&] { h->enc.finalize_weights((cudaStream_t)stream); });
}

CFGPP_API int cfgpp_clip_vision_encode(cfgpp_clip_vision_handle* h, const void* pixels, int dtype, int batch,
                                       void* embeds_out, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "pixel values: fp16 or fp32");
    h->enc.encode(pixels, dtype == CFGPP_F16, batch, (__half*)embeds_out, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_clip_vision_encode_hidden(cfgpp_clip_vision_handle* h, const void* pixels, int dtype, int batch,
                                              int skip, void* hidden_out, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "pixel values: fp16 or fp32");
    h->enc.encode_hidden(pixels, dtype == CFGPP_F16, batch, skip, (__half*)hidden_out, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_clip_vision_stats(cfgpp_clip_vision_handle* h, double* flops, size_t* workspace_bytes) {
  return guarded([&] {
    if (flops) *flops = h->enc.flops();
    if (workspace_bytes) *workspace_bytes = h->enc.workspace_bytes();
  });
}

// ---- operator-level entry points (one kernel launch each, on the caller's stream) ----
CFGPP_API int cfgpp_op_clip_embed(const int32_t* ids, const void* tok, const void* pos, void* out, int M, int T, int D,
                                  int vocab, void* stream) {
  return guarded([&] {
    run_clip_embed(ids, (const __half*)tok, (const __half*)pos, (__half*)out, M, T, D, vocab, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_clip_attention(const void* qkv, void* out, int B, int T, int heads, int D, void* stream) {
  return guarded([&] { run_clip_attention((const __half*)qkv, (__half*)out, B, T, heads, D, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_op_clip_activation(void* x, size_t n, int mode, void* stream) {
  return guarded([&] { run_clip_activation((__half*)x, n, mode, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_op_clip_gather_rows(const void* x, const int32_t* index, void* out, int B, int T, int D,
                                        void* stream) {
  return guarded([&] {
    run_clip_gather_rows((const __half*)x, index, (__half*)out, B, T, D, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_clip_patchify(const void* image, int dtype, void* out, int B, int S, int P, int Kp,
                                     void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "image: fp16 or fp32");
    CFGPP_REQUIRE(P >= 1 && S % P == 0 && Kp >= 3 * P * P, "image size a multiple of the patch, Kp >= 3 P P");
    run_clip_patchify(image, dtype == CFGPP_F16, (__half*)out, B, S, P, Kp, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_clip_vision_embed(const void* pe, const void* cls, const void* pos, void* out, int B, int np,
                                         int D, void* stream) {
  return guarded([&] {
    run_clip_vision_embed((const __half*)pe, (const __half*)cls, (const __half*)pos, (__half*)out, B, np, D,
                          (cudaStream_t)stream);
  });
}

}  // extern "C"
