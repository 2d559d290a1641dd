// cfgpp_b200 — IP-Adapter Plus image projection (diffusers IPAdapterPlusImageProjection, the Perceiver "Resampler") in
// the UNet handle's ip_plan_: the vision tower's penultimate hidden states [NB][T][E] -> Q image tokens [NB * Q][D].
// Host-side orchestration only: the GEMMs are gemm.cu's (residual adds in the epilogue), the attention is the head-dim-64
// flash kernel, the LayerNorms are norm.cu's (the two per layer in one launch) and GELU is the CLIP towers' erf mode.
#include "text_encoder.cuh"
#include "unet.cuh"

namespace cfgpp {

namespace {
std::string shape_str(const std::vector<int64_t>& s) {
  std::string o = "[";
  for (size_t i = 0; i < s.size(); ++i) o += (i ? ", " : "") + std::to_string(s[i]);
  return o + "]";
}
}  // namespace

// Every Resampler weight of geometry r, by its exact shape. Attach checks them, and so does every plan build: a key
// loaded again after attach may have another shape, and the plan's launches read the sizes r implies.
void Unet::require_resampler_weights(const cfgpp_ip_resampler_desc& r) const {
  const int64_t Q = r.num_queries, E = r.embed_dim, dim = r.dim, inner = 64 * r.heads, F = r.ff_mult * dim,
                D = d_.cross_attention_dim;
  CFGPP_REQUIRE(D % 8 == 0 && D <= 2048, "norm_out needs cross_attention_dim % 8 == 0 and <= 2048");
  auto need = [&](const std::string& key, std::vector<int64_t> shape) {
    CFGPP_REQUIRE(weights_.has(key), key + ": missing (load it with cfgpp_ip_adapter_load_weight first)");
    const std::vector<int64_t>& got = weights_.raw(key).shape;
    CFGPP_REQUIRE(got == shape, key + ": shape " + shape_str(got) + " does not fit the Resampler, expected " +
                                    shape_str(shape));
  };
  const std::string p = "image_proj.";
  need(p + "latents", {1, Q, dim});
  need(p + "proj_in.weight", {dim, E});
  need(p + "proj_in.bias", {dim});
  need(p + "proj_out.weight", {D, dim});
  need(p + "proj_out.bias", {D});
  need(p + "norm_out.weight", {D});
  need(p + "norm_out.bias", {D});
  for (int i = 0; i < r.depth; ++i) {
    const std::string l = p + "layers." + std::to_string(i) + ".";
    for (const char* n : {"0.norm1.", "0.norm2.", "1.0."}) {
      need(l + n + "weight", {dim});
      need(l + n + "bias", {dim});
    }
    need(l + "0.to_q.weight", {inner, dim});
    need(l + "0.to_kv.weight", {2 * inner, dim});
    need(l + "0.to_out.weight", {dim, inner});
    need(l + "1.1.weight", {F, dim});
    need(l + "1.3.weight", {dim, F});
  }
}

void Unet::ip_attach_resampler(const cfgpp_ip_resampler_desc& r) {
  CFGPP_REQUIRE(!is_cn_, "an IP-Adapter attaches to a UNet handle, not a ControlNet");
  CFGPP_REQUIRE(finalized_, "call cfgpp_finalize_weights first");
  CFGPP_REQUIRE(r.num_queries >= 1 && r.num_queries <= 64, "a Resampler has 1..64 queries (image tokens)");
  CFGPP_REQUIRE(r.embed_dim >= 64 && r.embed_dim % 64 == 0, "the hidden-state width E must be a positive multiple of 64");
  CFGPP_REQUIRE(r.seq_len >= 1 && r.seq_len <= 4096, "seq_len must be 1..4096 (ViT-H/14 at 224: 257)");
  CFGPP_REQUIRE(r.dim >= 64 && r.dim % 64 == 0 && r.dim <= 2048, "the Resampler width must be a multiple of 64, <= 2048");
  CFGPP_REQUIRE(r.heads >= 1 && r.heads <= 64, "the Resampler has 1..64 heads of 64");
  CFGPP_REQUIRE(r.depth >= 1 && r.depth <= 64, "the Resampler has 1..64 layers");
  CFGPP_REQUIRE(r.ff_mult >= 1 && r.ff_mult <= 16, "ff_mult must be 1..16");
  require_resampler_weights(r);
  ip_attach(r.num_queries, r.embed_dim);
  ip_rs_ = r;
}

void Unet::set_ip_image_hidden_states(const __half* hidden, cudaStream_t stream) {
  CFGPP_REQUIRE(ip_rs_.num_queries > 0, ip_ntok_ > 0 ? "the attached IP-Adapter takes image embeds "
                                                       "(cfgpp_set_ip_image_embeds), not hidden states"
                                                     : "no IP-Adapter attached");
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(hidden != nullptr, "null hidden states");
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(ip_hidden_, hidden,
                                   static_cast<size_t>(NB_) * ip_rs_.seq_len * ip_rs_.embed_dim * sizeof(__half),
                                   cudaMemcpyDeviceToDevice, stream));
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  run_plan(ip_plan_, stream);
  ip_ready_ = true;
}

void Unet::run_image_proj(__half* tokens_out, cudaStream_t stream) {
  CFGPP_REQUIRE(ip_ntok_ > 0 && ip_ready_, "no image projected for the prepared plan");
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  for (const auto& st : ip_plan_)
    if (st.name.rfind("image_proj.", 0) == 0) st.fn(stream);
  if (tokens_out)
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(tokens_out, ip_tokens_,
                                     static_cast<size_t>(NB_) * ip_ntok_ * d_.cross_attention_dim * sizeof(__half),
                                     cudaMemcpyDeviceToDevice, stream));
}

// x = proj_in(h); lat = latents per image; per layer: kv_in = [LN0(x), LN1(lat)], q_in = LN1(lat),
// lat += to_out(SDPA(to_q(q_in), to_kv(kv_in))), lat += W2 gelu(W1 LN_ff(lat)); tokens = norm_out(proj_out(lat)).
void Unet::build_ip_resampler() {
  const cfgpp_ip_resampler_desc r = ip_rs_;
  require_resampler_weights(r);
  const int NB = NB_, T = r.seq_len, Q = r.num_queries, E = r.embed_dim, dim = r.dim, heads = r.heads,
            inner = 64 * heads, F = r.ff_mult * dim, D = d_.cross_attention_dim, S = T + Q;
  const float eps = 1e-5f;
  const size_t sdim = dim;
  ip_hidden_ = alloc_act(static_cast<size_t>(NB) * T * E);
  __half* x = alloc_act(static_cast<size_t>(NB) * T * sdim);
  __half* lat = alloc_act(static_cast<size_t>(NB) * Q * sdim);
  __half* kv_in = alloc_act(static_cast<size_t>(NB) * S * sdim);
  __half* q_in = alloc_act(static_cast<size_t>(NB) * Q * sdim);  // also LN_ff's output
  __half* qb = alloc_act(static_cast<size_t>(NB) * Q * inner);
  __half* kv = alloc_act(static_cast<size_t>(NB) * S * 2 * inner);
  __half* o = alloc_act(static_cast<size_t>(NB) * Q * inner);
  __half* ffh = alloc_act(static_cast<size_t>(NB) * Q * F);
  __half* po = alloc_act(static_cast<size_t>(NB) * Q * D);
  const std::string p = "image_proj.";
  add_gemm(p + "proj_in", make_linear_op(ip_hidden_, E, nullptr, 0, 0, weights_.plain(p + "proj_in.weight"), NB * T, dim,
                                         E, weights_.plain(p + "proj_in.bias"), nullptr, 0, 1, x, dim, false));
  const __half* latents = weights_.plain(p + "latents");
  add_step(p + "latents", [=](cudaStream_t st) { run_copy_rows(latents, Q, dim, lat, dim, 0, NB * Q, st); });
  for (int i = 0; i < r.depth; ++i) {
    const std::string l = p + "layers." + std::to_string(i) + ".";
    const __half *g0 = weights_.plain(l + "0.norm1.weight"), *b0 = weights_.plain(l + "0.norm1.bias");
    const __half *g1 = weights_.plain(l + "0.norm2.weight"), *b1 = weights_.plain(l + "0.norm2.bias");
    add_step(l + "0.norm1+norm2", [=](cudaStream_t st) {
      run_ln_concat(x, lat, NB, T, Q, dim, g0, b0, g1, b1, eps, kv_in, q_in, st);
    });
    add_gemm(l + "0.to_q", make_linear_op(q_in, dim, nullptr, 0, 0, weights_.plain(l + "0.to_q.weight"), NB * Q, inner,
                                          dim, nullptr, nullptr, 0, 1, qb, inner, false));
    // k in the first inner columns, v in the second: the attention reads both in place with ld = 2 * inner
    add_gemm(l + "0.to_kv", make_linear_op(kv_in, dim, nullptr, 0, 0, weights_.plain(l + "0.to_kv.weight"), NB * S,
                                           2 * inner, dim, nullptr, nullptr, 0, 1, kv, 2 * inner, false));
    add_attn(l + "0.sdpa", make_attn_op(qb, inner, kv, 2 * inner, kv + inner, 2 * inner, o, inner, NB, heads, Q, S, 64));
    add_gemm(l + "0.to_out", make_linear_op(o, inner, nullptr, 0, 0, weights_.plain(l + "0.to_out.weight"), NB * Q, dim,
                                            inner, nullptr, lat, dim, 1, lat, dim, false));
    const __half *gf = weights_.plain(l + "1.0.weight"), *bf = weights_.plain(l + "1.0.bias");
    add_step(l + "1.0", [=](cudaStream_t st) { run_layernorm(lat, NB * Q, dim, gf, bf, eps, q_in, st); });
    add_gemm(l + "1.1", make_linear_op(q_in, dim, nullptr, 0, 0, weights_.plain(l + "1.1.weight"), NB * Q, F, dim,
                                       nullptr, nullptr, 0, 1, ffh, F, false));
    add_step(l + "1.2.gelu", [=](cudaStream_t st) { run_clip_activation(ffh, static_cast<size_t>(NB) * Q * F, 1, st); });
    add_gemm(l + "1.3", make_linear_op(ffh, F, nullptr, 0, 0, weights_.plain(l + "1.3.weight"), NB * Q, dim, F, nullptr,
                                       lat, dim, 1, lat, dim, false));
  }
  add_gemm(p + "proj_out", make_linear_op(lat, dim, nullptr, 0, 0, weights_.plain(p + "proj_out.weight"), NB * Q, D, dim,
                                          weights_.plain(p + "proj_out.bias"), nullptr, 0, 1, po, D, false));
  const __half *gn = weights_.plain(p + "norm_out.weight"), *bn = weights_.plain(p + "norm_out.bias");
  __half* tokens = ip_tokens_;
  add_step(p + "norm_out", [=](cudaStream_t st) { run_layernorm(po, NB * Q, D, gn, bn, eps, tokens, st); });
}

}  // namespace cfgpp
