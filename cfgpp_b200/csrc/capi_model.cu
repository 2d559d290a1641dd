// cfgpp_b200 — C ABI, model-level entry points (handle lifetime, weights, conditioning, forward, fused steps).
#include "capi_util.h"
#include "unet.cuh"

#include <algorithm>
#include <cstddef>
#include <cstring>

using namespace cfgpp;

struct cfgpp_handle {
  Unet unet;
  cfgpp_handle(const cfgpp_model_desc& d, int device, const cfgpp_controlnet_desc* cn = nullptr)
      : unet(d, device, cn) {}
};

namespace {
// The entry points that run, schedule or configure a UNet: a ControlNet handle runs only through the UNet it is
// attached to, so these refuse it with an error status instead of touching buffers it does not own.
Unet& unet_of(cfgpp_handle* h) {
  CFGPP_REQUIRE(h != nullptr, "null handle");
  CFGPP_REQUIRE(!h->unet.is_controlnet(), "this is a ControlNet handle: it runs through the UNet handle it is attached "
                                          "to (cfgpp_attach_controlnet)");
  return h->unet;
}
}  // namespace

extern "C" {

CFGPP_API int cfgpp_create_ex(const cfgpp_model_desc* desc, size_t desc_bytes, int device, cfgpp_handle** out) {
  return guarded([&] {
    CFGPP_REQUIRE(desc && out, "null argument");
    constexpr size_t legacy = offsetof(cfgpp_model_desc, prediction_type);
    CFGPP_REQUIRE(desc_bytes == legacy || desc_bytes == sizeof(cfgpp_model_desc), "unknown cfgpp_model_desc size");
    cfgpp_model_desc d{};  // fields the caller's layout does not have stay 0 (prediction_type: epsilon)
    memcpy(&d, desc, desc_bytes);
    *out = new cfgpp_handle(d, device);
  });
}

CFGPP_API int cfgpp_create(const cfgpp_model_desc* desc, int device, cfgpp_handle** out) {
  return cfgpp_create_ex(desc, offsetof(cfgpp_model_desc, prediction_type), device, out);
}

CFGPP_API int cfgpp_destroy(cfgpp_handle* h) {
  return guarded([&] { delete h; });
}

CFGPP_API int cfgpp_load_weight(cfgpp_handle* h, const char* key, const void* data, const int64_t* shape, int ndim,
                                int dtype, void* stream) {
  return guarded([&] { h->unet.load_weight(key, data, shape, ndim, dtype, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_finalize_weights(cfgpp_handle* h, void* stream) {
  return guarded([&] { h->unet.finalize_weights((cudaStream_t)stream); });
}

CFGPP_API int cfgpp_lora_add(cfgpp_handle* h, int adapter, const char* key, const void* down, const void* up, int rank,
                             float alpha, int dtype, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(key, "null key");
    unet_of(h).lora_add(adapter, key, down, up, rank, alpha, dtype, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_lora_set_scales(cfgpp_handle* h, const float* scales_host, int n_adapters, void* stream) {
  return guarded([&] { unet_of(h).lora_set_scales(scales_host, n_adapters, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_lora_clear(cfgpp_handle* h, void* stream) {
  return guarded([&] { unet_of(h).lora_clear((cudaStream_t)stream); });
}

CFGPP_API int cfgpp_lora_stats(cfgpp_handle* h, int* n_adapters, int* n_targets, size_t* backup_bytes,
                               size_t* bytes_moved) {
  return guarded([&] { h->unet.lora_stats(n_adapters, n_targets, backup_bytes, bytes_moved); });
}

CFGPP_API int cfgpp_prepare(cfgpp_handle* h, int batch, int h_lat, int w_lat) {
  return guarded([&] { unet_of(h).prepare(batch, h_lat, w_lat); });
}

CFGPP_API int cfgpp_workspace_bytes(cfgpp_handle* h, size_t* bytes) {
  return guarded([&] { *bytes = h->unet.workspace_bytes(); });
}

CFGPP_API int cfgpp_forward_flops(cfgpp_handle* h, double* flops) {
  return guarded([&] { *flops = h->unet.forward_flops(); });
}

CFGPP_API int cfgpp_launches_per_step(cfgpp_handle* h, int* n) {
  return guarded([&] { *n = h->unet.launches_per_step(); });
}

CFGPP_API int cfgpp_plan_stats(cfgpp_handle* h, double* step_flops, double* prompt_flops, int* prompt_launches) {
  return guarded([&] {
    if (step_flops) *step_flops = h->unet.forward_flops() - h->unet.prompt_flops();
    if (prompt_flops) *prompt_flops = h->unet.prompt_flops();
    if (prompt_launches) *prompt_launches = h->unet.prompt_launches();
  });
}

CFGPP_API int cfgpp_set_prompt(cfgpp_handle* h, const void* ctx, int n_ctx, const void* pooled, const float* time_ids,
                               int add_rows, void* stream) {
  return guarded([&] {
    unet_of(h).set_prompt((const __half*)ctx, n_ctx, (const __half*)pooled, time_ids, add_rows, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_unet_forward(cfgpp_handle* h, const void* z, int z_dtype, float t, float in_scale, void* eps_uc,
                                 void* eps_c, void* stream) {
  return guarded([&] {
    unet_of(h).unet_forward(z, z_dtype, t, in_scale, (__half*)eps_uc, (__half*)eps_c, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_set_schedule(cfgpp_handle* h, int method, int state_dtype, const cfgpp_step_state* steps,
                                 int nsteps, void* stream) {
  return guarded([&] { unet_of(h).set_schedule(method, state_dtype, steps, nsteps, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_set_state(cfgpp_handle* h, const void* z, int z_dtype, void* stream) {
  return guarded([&] { unet_of(h).set_state(z, z_dtype, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_set_noise(cfgpp_handle* h, const void* noise_dev, int slots, void* stream) {
  return guarded([&] { unet_of(h).set_noise((const __half*)noise_dev, slots, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_set_guidance(cfgpp_handle* h, const float* lambda_host, int n, void* stream) {
  return guarded([&] { unet_of(h).set_guidance(lambda_host, n, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_set_v_coefs(cfgpp_handle* h, const float* ab_host, int nsteps, void* stream) {
  return guarded([&] { unet_of(h).set_v_coefs(ab_host, nsteps, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_run_steps(cfgpp_handle* h, int first_step, int nsteps, void* stream) {
  return guarded([&] { unet_of(h).run_steps(first_step, nsteps, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_get_state(cfgpp_handle* h, int which, void* out, void* stream) {
  return guarded([&] { unet_of(h).get_state(which, out, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_apply_step(cfgpp_handle* h, int step, const void* eps_uc, const void* eps_c, void* stream) {
  return guarded([&] { unet_of(h).apply_step(step, (const __half*)eps_uc, (const __half*)eps_c, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_profile_forward(cfgpp_handle* h, const void* z, int z_dtype, float t, float in_scale, int max_n,
                                    int* n_out, float* ms_out, double* flops_out, int* kind_out, char* names_out,
                                    int name_stride, void* stream) {
  return guarded([&] {
    auto prof = unet_of(h).profile_forward(z, z_dtype, t, in_scale, (cudaStream_t)stream);
    const int n = static_cast<int>(prof.size()) < max_n ? static_cast<int>(prof.size()) : max_n;
    *n_out = n;
    for (int i = 0; i < n; ++i) {
      ms_out[i] = prof[i].ms;
      flops_out[i] = prof[i].flops;
      kind_out[i] = prof[i].kind;
      if (names_out && name_stride > 0) {
        const size_t len = std::min<size_t>(prof[i].name.size(), static_cast<size_t>(name_stride - 1));
        memcpy(names_out + static_cast<size_t>(i) * name_stride, prof[i].name.data(), len);
        names_out[static_cast<size_t>(i) * name_stride + len] = 0;
      }
    }
  });
}

CFGPP_API int cfgpp_controlnet_create(const cfgpp_controlnet_desc* desc, int device, cfgpp_handle** out) {
  return guarded([&] {
    CFGPP_REQUIRE(desc && out, "null argument");
    *out = new cfgpp_handle(desc->model, device, desc);
  });
}

CFGPP_API int cfgpp_attach_controlnet(cfgpp_handle* h, cfgpp_handle* cn) {
  return guarded([&] { unet_of(h).attach_controlnet(cn ? &cn->unet : nullptr); });
}

CFGPP_API int cfgpp_set_control_image(cfgpp_handle* h, const void* image, int dtype, void* stream) {
  return guarded([&] { unet_of(h).set_control_image(image, dtype, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_set_control_scale(cfgpp_handle* h, float scale, void* stream) {
  return guarded([&] { unet_of(h).set_control_scale(scale, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_set_control_scales(cfgpp_handle* h, const float* scales_host, int nsteps, void* stream) {
  return guarded([&] { unet_of(h).set_control_scales(scales_host, nsteps, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_ip_adapter_load_weight(cfgpp_handle* h, const char* key, const void* data, const int64_t* shape,
                                           int ndim, int dtype, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(key && data && shape, "null argument");
    unet_of(h).ip_load_weight(key, data, shape, ndim, dtype, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_ip_adapter_attach(cfgpp_handle* h, int n_tokens, int image_embed_dim) {
  return guarded([&] {
    CFGPP_REQUIRE(n_tokens >= 1, "an IP-Adapter has at least one image token (cfgpp_ip_adapter_clear detaches)");
    unet_of(h).ip_attach(n_tokens, image_embed_dim);
  });
}

CFGPP_API int cfgpp_ip_adapter_clear(cfgpp_handle* h) {
  return guarded([&] { unet_of(h).ip_attach(0, 0); });
}

CFGPP_API int cfgpp_set_ip_image_embeds(cfgpp_handle* h, const void* embeds_dev, void* stream) {
  return guarded([&] { unet_of(h).set_ip_image_embeds((const __half*)embeds_dev, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_ip_adapter_attach_resampler(cfgpp_handle* h, const cfgpp_ip_resampler_desc* desc) {
  return guarded([&] {
    CFGPP_REQUIRE(desc != nullptr, "null argument");
    unet_of(h).ip_attach_resampler(*desc);
  });
}

CFGPP_API int cfgpp_set_ip_image_hidden_states(cfgpp_handle* h, const void* hidden_dev, void* stream) {
  return guarded([&] { unet_of(h).set_ip_image_hidden_states((const __half*)hidden_dev, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_set_ip_adapter_scale(cfgpp_handle* h, float scale, void* stream) {
  return guarded([&] { unet_of(h).set_ip_scale(scale, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_t2i_attach(cfgpp_handle* h, int n_features) {
  return guarded([&] { unet_of(h).t2i_attach(n_features); });
}

CFGPP_API int cfgpp_set_t2i_features(cfgpp_handle* h, const void* const* features_dev, void* stream) {
  return guarded([&] {
    unet_of(h).set_t2i_features(reinterpret_cast<const __half* const*>(features_dev), (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_set_t2i_active(cfgpp_handle* h, int on, void* stream) {
  return guarded([&] { unet_of(h).set_t2i_active(on, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_set_t2i_steps(cfgpp_handle* h, const int* on_host, int nsteps, void* stream) {
  return guarded([&] { unet_of(h).set_t2i_steps(on_host, nsteps, (cudaStream_t)stream); });
}

// Debug aid (not in the public header): how many step graphs the handle has captured.
CFGPP_API int cfgpp_dbg_graph_captures(cfgpp_handle* h, int* n) {
  return guarded([&] { *n = unet_of(h).graph_captures(); });
}

// Test and measurement aid (not in the public header): the IP-Adapter image projection alone, on the rows the last
// cfgpp_set_ip_image_embeds / cfgpp_set_ip_image_hidden_states set, and its tokens [2*batch * n_tokens, D] fp16
// copied into tokens_out_dev (may be null).
CFGPP_API int cfgpp_dbg_ip_image_proj(cfgpp_handle* h, void* tokens_out_dev, void* stream) {
  return guarded([&] { unet_of(h).run_image_proj((__half*)tokens_out_dev, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_controlnet_embed(cfgpp_handle* cn, const void* image, int dtype, int batch, int height, int width,
                                     void* out, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "control image: fp16 or fp32 tensor");
    cn->unet.cond_embed(image, dtype == CFGPP_F16, batch, height, width, (__half*)out, (cudaStream_t)stream);
  });
}

}  // extern "C"
