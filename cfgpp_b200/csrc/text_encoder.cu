// cfgpp_b200 — CLIP text tower executor (see text_encoder.cuh). Host-side orchestration only.
#include "text_encoder.cuh"

#include <algorithm>
#include <cmath>

namespace cfgpp {

void gemm_configure();

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
  const size_t D = d_.hidden_size;
  const std::string tm = "text_model.";
  // q | k | v projections of a layer as one [3D][D] operand (one GEMM instead of three)
  for (int l = 0; l < d_.num_layers; ++l) {
    const std::string a = tm + "encoder.layers." + std::to_string(l) + ".self_attn.";
    __half* w = weights_.alloc(3 * D * D);
    __half* b = weights_.alloc(3 * D);
    const char* names[3] = {"q_proj", "k_proj", "v_proj"};
    for (int i = 0; i < 3; ++i) {
      CFGPP_CHECK_CUDA(cudaMemcpyAsync(w + i * D * D, weights_.plain(a + names[i] + ".weight", D * D), D * D * sizeof(__half),
                                       cudaMemcpyDeviceToDevice, stream));
      CFGPP_CHECK_CUDA(cudaMemcpyAsync(b + i * D, weights_.plain(a + names[i] + ".bias", D), D * sizeof(__half),
                                       cudaMemcpyDeviceToDevice, stream));
    }
    qkv_w_.push_back(w);
    qkv_b_.push_back(b);
  }
  CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));
  finalized_ = true;
  try {  // structural validation: building a plan touches (and size-checks) every weight
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
  const float eps = d_.layer_norm_eps;
  const int heads = d_.num_heads, act_mode = d_.hidden_act;
  __half *x0 = x0_, *x1 = x1_, *ln = ln_, *qkv = qkv_, *att = att_, *mlp = mlp_;
  for (int l = 0; l < d_.num_layers; ++l) {
    const std::string p = tm + "encoder.layers." + std::to_string(l) + ".";
    std::vector<Step> steps;
    auto add_gemm = [&](const GemmOp& op) {
      flops_ += op.flops();
      steps.push_back([op](cudaStream_t st) { run_gemm_op(op, st); });
    };
    const __half *g1 = weights_.plain(p + "layer_norm1.weight", sD), *b1 = weights_.plain(p + "layer_norm1.bias", sD);
    const __half *g2 = weights_.plain(p + "layer_norm2.weight", sD), *b2 = weights_.plain(p + "layer_norm2.bias", sD);
    // x1 = x0 + out_proj(attention(q, k, v of LN1(x0)))
    steps.push_back([=](cudaStream_t st) { run_layernorm(x0, M, D, g1, b1, eps, ln, st); });
    add_gemm(make_linear_op(ln, D, nullptr, 0, 0, qkv_w_[l], M, 3 * D, D, qkv_b_[l], nullptr, 0, 1, qkv, 3 * D, false));
    steps.push_back([=](cudaStream_t st) { run_clip_attention(qkv, att, NB, T, heads, D, st); });
    flops_ += 2.0 * NB * heads * static_cast<double>(T) * T * 64.0;  // causal: half of 2 * (QK^T + PV)
    add_gemm(make_linear_op(att, D, nullptr, 0, 0, weights_.plain(p + "self_attn.out_proj.weight", sD * sD), M, D, D,
                            weights_.plain(p + "self_attn.out_proj.bias", sD), x0, D, 1, x1, D, false));
    // x0 = x1 + fc2(act(fc1(LN2(x1))))
    steps.push_back([=](cudaStream_t st) { run_layernorm(x1, M, D, g2, b2, eps, ln, st); });
    add_gemm(make_linear_op(ln, D, nullptr, 0, 0, weights_.plain(p + "mlp.fc1.weight", sI * sD), M, I, D,
                            weights_.plain(p + "mlp.fc1.bias", sI), nullptr, 0, 1, mlp, I, false));
    steps.push_back([=](cudaStream_t st) { run_clip_activation(mlp, static_cast<size_t>(M) * I, act_mode, st); });
    add_gemm(make_linear_op(mlp, I, nullptr, 0, 0, weights_.plain(p + "mlp.fc2.weight", sD * sI), M, D, I,
                            weights_.plain(p + "mlp.fc2.bias", sD), x1, D, 1, x0, D, false));
    layer_plan_.push_back(std::move(steps));
  }
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

}  // namespace cfgpp
