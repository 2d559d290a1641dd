// cfgpp_b200 — CLIP text tower executor (see text_encoder.cuh). Host-side orchestration only.
#include "text_encoder.cuh"

#include <algorithm>
#include <cmath>

#include "attention.cuh"

namespace cfgpp {

void gemm_configure();
void attn_configure();

std::vector<std::vector<ClipStep>> build_clip_layers(const ClipLayerArgs& a, double* flops) {
  const int D = a.D, I = a.I, M = a.M, act_mode = a.act_mode;
  const size_t sD = D, sI = I;
  const float eps = a.eps;
  __half *x0 = a.x0, *x1 = a.x1, *ln = a.ln, *qkv = a.qkv, *att = a.att, *mlp = a.mlp;
  const int hd = D / a.heads, qkv_n = 3 * a.heads * a.hdp, att_c = a.heads * a.hdp;
  WeightStore& w = *a.weights;
  std::vector<std::vector<ClipStep>> plan;
  for (int l = 0; l < a.layers; ++l) {
    const std::string p = a.prefix + std::to_string(l) + ".";
    const std::string q = p + "self_attn.q_proj", k = p + "self_attn.k_proj", v = p + "self_attn.v_proj",
                      o = p + "self_attn.out_proj.weight";
    for (const std::string& n : {q, k, v}) {  // sizes are checked before anything is packed from them
      w.plain(n + ".weight", sD * sD);
      w.plain(n + ".bias", sD);
    }
    w.plain(o, sD * sD);
    // q | k | v as one operand (one GEMM instead of three) with every head zero-padded to hdp rows, and out_proj with
    // hdp-wide head columns
    const __half* qkv_w = w.packed_heads_rows({q + ".weight", k + ".weight", v + ".weight"}, a.heads, hd, a.hdp);
    const __half* qkv_b = w.packed_heads_rows({q + ".bias", k + ".bias", v + ".bias"}, a.heads, hd, a.hdp);
    const __half* out_w = w.packed_heads_cols(o, a.heads, hd, a.hdp);
    std::vector<ClipStep> steps;
    auto add_gemm = [&](const GemmOp& op) {
      *flops += op.flops();
      steps.push_back([op](cudaStream_t st) { run_gemm_op(op, st); });
    };
    const __half *g1 = w.plain(p + "layer_norm1.weight", sD), *b1 = w.plain(p + "layer_norm1.bias", sD);
    const __half *g2 = w.plain(p + "layer_norm2.weight", sD), *b2 = w.plain(p + "layer_norm2.bias", sD);
    // x1 = x0 + out_proj(attention(q, k, v of LN1(x0)))
    steps.push_back([=](cudaStream_t st) { run_layernorm(x0, M, D, g1, b1, eps, ln, st); });
    add_gemm(make_linear_op(ln, D, nullptr, 0, 0, qkv_w, M, qkv_n, D, qkv_b, nullptr, 0, 1, qkv, qkv_n, false));
    const auto attention = a.attention;
    steps.push_back([=](cudaStream_t st) { attention(qkv, att, st); });
    *flops += a.attention_flops;
    add_gemm(make_linear_op(att, att_c, nullptr, 0, 0, out_w, M, D, att_c,
                            w.plain(p + "self_attn.out_proj.bias", sD), x0, D, 1, x1, D, false));
    // x0 = x1 + fc2(act(fc1(LN2(x1))))
    steps.push_back([=](cudaStream_t st) { run_layernorm(x1, M, D, g2, b2, eps, ln, st); });
    add_gemm(make_linear_op(ln, D, nullptr, 0, 0, w.plain(p + "mlp.fc1.weight", sI * sD), M, I, D,
                            w.plain(p + "mlp.fc1.bias", sI), nullptr, 0, 1, mlp, I, false));
    steps.push_back([=](cudaStream_t st) { run_clip_activation(mlp, static_cast<size_t>(M) * I, act_mode, st); });
    add_gemm(make_linear_op(mlp, I, nullptr, 0, 0, w.plain(p + "mlp.fc2.weight", sD * sI), M, D, I,
                            w.plain(p + "mlp.fc2.bias", sD), x1, D, 1, x0, D, false));
    plan.push_back(std::move(steps));
  }
  return plan;
}

ClipTextEncoder::ClipTextEncoder(const cfgpp_clip_desc& d, int device) : d_(d), device_(device), sk_(device) {
  CFGPP_CHECK_CUDA(cudaSetDevice(device));
  CFGPP_REQUIRE(d.vocab_size >= 2 && d.num_layers >= 1 && d.num_layers <= 64, "bad vocab_size / num_layers");
  CFGPP_REQUIRE(d.max_positions >= 1 && d.max_positions <= 128, "max_positions must be 1..128 (CLIP: 77)");
  CFGPP_REQUIRE(d.num_heads >= 1 && d.hidden_size == d.num_heads * 64, "hidden_size must be num_heads * 64");
  CFGPP_REQUIRE(d.intermediate_size % 64 == 0 && d.intermediate_size > 0, "intermediate_size must be a multiple of 64");
  CFGPP_REQUIRE(d.hidden_act == 0 || d.hidden_act == 1, "hidden_act: 0 quick_gelu, 1 gelu");
  CFGPP_REQUIRE(d.projection_dim >= 0 && d.projection_dim % 8 == 0, "projection_dim must be 0 or a multiple of 8");
  CFGPP_REQUIRE(d.layer_norm_eps > 0.f, "layer_norm_eps must be positive");
  gemm_configure();
}

void ClipTextEncoder::load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                                  cudaStream_t stream) {
  CFGPP_REQUIRE(!finalized_, "weights already finalized");
  weights_.load(key, data, shape, ndim, dtype, stream);
}

void ClipTextEncoder::finalize_weights(cudaStream_t stream) {
  CFGPP_REQUIRE(!finalized_, "weights already finalized");
  CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));
  finalized_ = true;
  try {  // structural validation: building a plan touches (size-checks and packs) every weight
    prepare(1, d_.max_positions);
  } catch (...) {
    finalized_ = false;
    throw;
  }
}

void ClipTextEncoder::prepare(int batch, int tokens) {
  CFGPP_REQUIRE(finalized_, "call cfgpp_clip_finalize_weights first");
  CFGPP_REQUIRE(batch >= 1 && batch <= 16, "encode batch must be 1..16 prompts");
  CFGPP_REQUIRE(tokens >= 1 && tokens <= d_.max_positions, "token count exceeds max_positions");
  CFGPP_CHECK_CUDA(cudaSetDevice(device_));
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  act_.clear();
  layer_plan_.clear();
  flops_ = 0.0;
  B_ = 0;
  const int D = d_.hidden_size, I = d_.intermediate_size, T = tokens, NB = batch, M = NB * T;
  const size_t sD = D, sI = I;
  auto act = [&](size_t numel) { return act_.alloc<__half>(numel); };
  x0_ = act(M * sD);
  x1_ = act(M * sD);
  ln_ = act(M * sD);
  qkv_ = act(M * 3 * sD);
  att_ = act(M * sD);
  mlp_ = act(M * sI);
  last_ = act(M * sD);
  pool_ = act(16 * sD);
  const std::string tm = "text_model.";
  weights_.plain(tm + "embeddings.token_embedding.weight", static_cast<size_t>(d_.vocab_size) * sD);
  weights_.plain(tm + "embeddings.position_embedding.weight", static_cast<size_t>(d_.max_positions) * sD);
  weights_.plain(tm + "final_layer_norm.weight", sD);
  weights_.plain(tm + "final_layer_norm.bias", sD);
  if (d_.projection_dim > 0) weights_.plain("text_projection.weight", static_cast<size_t>(d_.projection_dim) * sD);
  const int heads = d_.num_heads;
  ClipLayerArgs a{&weights_, tm + "encoder.layers.", d_.num_layers, D, I, M, d_.hidden_act, d_.layer_norm_eps, heads, 64,
                  nullptr, 2.0 * NB * heads * static_cast<double>(T) * T * 64.0,  // causal: half
                  x0_, x1_, ln_, qkv_, att_, mlp_};
  a.attention = [=](const __half* qkv, __half* att, cudaStream_t st) { run_clip_attention(qkv, att, NB, T, heads, D, st); };
  layer_plan_ = build_clip_layers(a, &flops_);
  B_ = NB;
  T_ = T;
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
}

void ClipTextEncoder::encode(const int* ids, const int* pooled_index, int batch, int tokens, int skip,
                             __half* hidden_out, __half* last_out, __half* pooled_out, cudaStream_t stream) {
  CFGPP_REQUIRE(ids != nullptr, "null input_ids");
  CFGPP_REQUIRE(skip >= 0 && skip <= d_.num_layers, "skip must be 0..num_layers (hidden_states[num_layers - skip])");
  CFGPP_REQUIRE(pooled_out == nullptr || pooled_index != nullptr, "pooled output requested without pooled_index");
  if (batch != B_ || tokens != T_) prepare(batch, tokens);
  const int D = d_.hidden_size, M = batch * tokens;
  const std::string tm = "text_model.";
  run_clip_embed(ids, weights_.plain(tm + "embeddings.token_embedding.weight"), weights_.plain(tm + "embeddings.position_embedding.weight"),
                 x0_, M, tokens, D, d_.vocab_size, stream);
  const bool need_last = last_out != nullptr || pooled_out != nullptr;
  const int wanted = d_.num_layers - skip;  // index into hidden_states
  const int run_layers = need_last ? d_.num_layers : (hidden_out ? wanted : 0);
  const size_t bytes = static_cast<size_t>(M) * D * sizeof(__half);
  if (hidden_out && wanted == 0)
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(hidden_out, x0_, bytes, cudaMemcpyDeviceToDevice, stream));
  for (int l = 0; l < run_layers; ++l) {
    for (auto& fn : layer_plan_[l]) fn(stream);
    if (hidden_out && wanted == l + 1)
      CFGPP_CHECK_CUDA(cudaMemcpyAsync(hidden_out, x0_, bytes, cudaMemcpyDeviceToDevice, stream));
  }
  if (!need_last) return;
  __half* last = last_out ? last_out : last_;
  run_layernorm(x0_, M, D, weights_.plain(tm + "final_layer_norm.weight"), weights_.plain(tm + "final_layer_norm.bias"), d_.layer_norm_eps,
                last, stream);
  if (pooled_out) {
    if (d_.projection_dim > 0) {
      run_clip_gather_rows(last, pooled_index, pool_, batch, tokens, D, stream);
      run_small_linear(pool_, D, weights_.plain("text_projection.weight"), nullptr, nullptr, 0, pooled_out, d_.projection_dim,
                       nullptr, batch, d_.projection_dim, D, false, stream);
    } else {
      run_clip_gather_rows(last, pooled_index, pooled_out, batch, tokens, D, stream);
    }
  }
}


// ------------------------------------------------------------------------------------------------------------
// vision tower
// ------------------------------------------------------------------------------------------------------------
ClipVisionEncoder::ClipVisionEncoder(const cfgpp_clip_vision_desc& d, int device) : d_(d), device_(device), sk_(device) {
  CFGPP_CHECK_CUDA(cudaSetDevice(device));
  CFGPP_REQUIRE(d.num_layers >= 1 && d.num_layers <= 64, "num_layers must be 1..64");
  CFGPP_REQUIRE(d.num_heads >= 1 && d.hidden_size % d.num_heads == 0 && d.hidden_size / d.num_heads <= 192 &&
                    d.hidden_size % 64 == 0,
                "hidden_size must be num_heads * head_dim with head_dim <= 192, a multiple of 64");
  CFGPP_REQUIRE(d.intermediate_size % 64 == 0 && d.intermediate_size > 0, "intermediate_size must be a multiple of 64");
  CFGPP_REQUIRE(d.patch_size >= 1 && d.image_size % d.patch_size == 0, "image_size must be a multiple of patch_size");
  CFGPP_REQUIRE(d.hidden_act == 0 || d.hidden_act == 1, "hidden_act: 0 quick_gelu, 1 gelu");
  CFGPP_REQUIRE(d.projection_dim > 0 && d.projection_dim % 8 == 0, "projection_dim must be a positive multiple of 8");
  CFGPP_REQUIRE(d.layer_norm_eps > 0.f, "layer_norm_eps must be positive");
  np_ = (d.image_size / d.patch_size) * (d.image_size / d.patch_size);
  T_ = np_ + 1;
  Kp_ = (3 * d.patch_size * d.patch_size + 63) / 64 * 64;
  hdp_ = attn_padded_head_dim(d.hidden_size / d.num_heads);
  Cp_ = d.num_heads * hdp_;
  gemm_configure();
  attn_configure();
}

void ClipVisionEncoder::load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                                    cudaStream_t stream) {
  CFGPP_REQUIRE(!finalized_, "weights already finalized");
  weights_.load(key, data, shape, ndim, dtype, stream);
}

void ClipVisionEncoder::finalize_weights(cudaStream_t stream) {
  CFGPP_REQUIRE(!finalized_, "weights already finalized");
  CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));
  // the patch conv as [D][Kp], K zero-padded to whole 64-wide k blocks
  const int K = 3 * d_.patch_size * d_.patch_size;
  const std::string patch = "vision_model.embeddings.patch_embedding.weight";
  weights_.plain(patch, static_cast<size_t>(d_.hidden_size) * K);
  patch_w_ = weights_.packed_heads_cols(patch, 1, K, Kp_);
  finalized_ = true;
  try {
    prepare(1);
  } catch (...) {
    finalized_ = false;
    throw;
  }
}

void ClipVisionEncoder::prepare(int batch) {
  CFGPP_REQUIRE(finalized_, "call cfgpp_clip_vision_finalize_weights first");
  CFGPP_REQUIRE(batch >= 1 && batch <= 16, "encode batch must be 1..16 images");
  CFGPP_CHECK_CUDA(cudaSetDevice(device_));
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  act_.clear();
  layer_plan_.clear();
  flops_ = 0.0;
  B_ = 0;
  const int D = d_.hidden_size, I = d_.intermediate_size, T = T_, NB = batch, M = NB * T, H = d_.num_heads;
  const int hd = D / H, Cp = Cp_;
  const size_t sD = D;
  auto act = [&](size_t numel) { return act_.alloc<__half>(numel); };
  patches_ = act(static_cast<size_t>(NB) * np_ * Kp_);
  pe_ = act(static_cast<size_t>(NB) * np_ * sD);
  emb_ = act(M * sD);
  x0_ = act(M * sD);
  x1_ = act(M * sD);
  ln_ = act(M * sD);
  qkv_ = act(static_cast<size_t>(M) * 3 * Cp);
  att_ = act(static_cast<size_t>(M) * Cp);
  mlp_ = act(static_cast<size_t>(M) * I);
  cls_ = act(NB * sD);
  cls_ln_ = act(NB * sD);
  const std::string vm = "vision_model.";
  weights_.plain(vm + "embeddings.class_embedding", sD);
  weights_.plain(vm + "embeddings.position_embedding.weight", static_cast<size_t>(T) * sD);
  for (const char* n : {"pre_layrnorm", "post_layernorm"}) {
    weights_.plain(vm + n + ".weight", sD);
    weights_.plain(vm + n + ".bias", sD);
  }
  weights_.plain("visual_projection.weight", static_cast<size_t>(d_.projection_dim) * sD);
  flops_ += 2.0 * NB * np_ * static_cast<double>(D) * 3 * d_.patch_size * d_.patch_size;
  ClipLayerArgs a{&weights_, vm + "encoder.layers.", d_.num_layers, D, I, M, d_.hidden_act, d_.layer_norm_eps, H, hdp_,
                  nullptr, 4.0 * NB * H * static_cast<double>(T) * T * hd, x0_, x1_, ln_, qkv_, att_, mlp_};
  const AttnOp op = make_attn_op(qkv_, 3 * Cp, qkv_ + Cp, 3 * Cp, qkv_ + 2 * Cp, 3 * Cp, att_, Cp, NB, H, T, T, hd);
  a.attention = [op](const __half*, __half*, cudaStream_t st) { run_attn_op(op, st); };
  layer_plan_ = build_clip_layers(a, &flops_);
  flops_ += 2.0 * NB * static_cast<double>(d_.projection_dim) * D;
  B_ = NB;
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
}

void ClipVisionEncoder::embed(const void* image, int is_half, int batch, cudaStream_t stream) {
  CFGPP_REQUIRE(image != nullptr, "null argument");
  if (batch != B_) prepare(batch);
  const int D = d_.hidden_size, M = batch * T_;
  const std::string vm = "vision_model.";
  run_clip_patchify(image, is_half, patches_, batch, d_.image_size, d_.patch_size, Kp_, stream);
  run_gemm_op(make_linear_op(patches_, Kp_, nullptr, 0, 0, patch_w_, batch * np_, D, Kp_, nullptr, nullptr, 0, 1, pe_, D,
                             false),
              stream);
  run_clip_vision_embed(pe_, weights_.plain(vm + "embeddings.class_embedding"),
                        weights_.plain(vm + "embeddings.position_embedding.weight"), emb_, batch, np_, D, stream);
  run_layernorm(emb_, M, D, weights_.plain(vm + "pre_layrnorm.weight"), weights_.plain(vm + "pre_layrnorm.bias"),
                d_.layer_norm_eps, x0_, stream);
}

void ClipVisionEncoder::encode(const void* image, int is_half, int batch, __half* embeds_out, cudaStream_t stream) {
  CFGPP_REQUIRE(embeds_out != nullptr, "null argument");
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  embed(image, is_half, batch, stream);
  const int D = d_.hidden_size;
  const std::string vm = "vision_model.";
  for (auto& layer : layer_plan_)
    for (auto& fn : layer) fn(stream);
  CFGPP_CHECK_CUDA(cudaMemcpy2DAsync(cls_, D * sizeof(__half), x0_, static_cast<size_t>(T_) * D * sizeof(__half),
                                     D * sizeof(__half), batch, cudaMemcpyDeviceToDevice, stream));
  run_layernorm(cls_, batch, D, weights_.plain(vm + "post_layernorm.weight"), weights_.plain(vm + "post_layernorm.bias"),
                d_.layer_norm_eps, cls_ln_, stream);
  run_small_linear(cls_ln_, D, weights_.plain("visual_projection.weight"), nullptr, nullptr, 0, embeds_out,
                   d_.projection_dim, nullptr, batch, d_.projection_dim, D, false, stream);
}

void ClipVisionEncoder::encode_hidden(const void* image, int is_half, int batch, int skip, __half* hidden_out,
                                      cudaStream_t stream) {
  CFGPP_REQUIRE(hidden_out != nullptr, "null argument");
  CFGPP_REQUIRE(skip >= 0 && skip <= d_.num_layers, "skip must be 0..num_layers (hidden_states[num_layers - skip])");
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  embed(image, is_half, batch, stream);
  // hidden_states[0] is pre_layrnorm's output; layer l writes hidden_states[l + 1]. The layers after the wanted one
  // do not run.
  for (int l = 0; l < d_.num_layers - skip; ++l)
    for (auto& fn : layer_plan_[l]) fn(stream);
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(hidden_out, x0_, static_cast<size_t>(batch) * T_ * d_.hidden_size * sizeof(__half),
                                   cudaMemcpyDeviceToDevice, stream));
}

}  // namespace cfgpp
