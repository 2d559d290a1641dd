// cfgpp_b200 — UNet2DConditionModel executor (see unet.cuh). Host-side orchestration only; every FLOP runs in the
// hand-written kernels of gemm.cu / attention.cu / norm.cu / elementwise.cu.
#include "unet.cuh"

#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace cfgpp {

void gemm_configure();
void attn_configure();

Unet::Unet(const cfgpp_model_desc& d, int device, const cfgpp_controlnet_desc* cn)
    : d_(d), device_(device), sk_(device) {
  CFGPP_CHECK_CUDA(cudaSetDevice(device));
  if (cn) {
    is_cn_ = true;
    cn_desc_ = *cn;
    CFGPP_REQUIRE(cn->conditioning_channels >= 1 && cn->conditioning_channels <= 64,
                  "conditioning_channels must be 1..64");
    CFGPP_REQUIRE(cn->num_embedding_levels == 4,
                  "the conditioning embedding must take 4 channel counts (it downsamples the image by 8 to the latent)");
    for (int i = 0; i < cn->num_embedding_levels; ++i)
      CFGPP_REQUIRE(cn->embedding_channels[i] >= 1, "conditioning embedding channels must be positive");
    CFGPP_REQUIRE(d.block_out_channels[0] % 8 == 0, "block_out_channels[0] must be a multiple of 8");
  }
  CFGPP_REQUIRE(d.num_levels >= 2 && d.num_levels <= CFGPP_MAX_LEVELS, "num_levels must be 2..4");
  CFGPP_REQUIRE(d.norm_num_groups == 32, "only GroupNorm(32) is implemented");
  CFGPP_REQUIRE(d.in_channels == 4 && d.out_channels == 4, "latent channels must be 4");
  time_embed_dim_ = d.block_out_channels[0] * 4;
  has_aug_ = d.addition_time_embed_dim > 0;
  if (has_aug_) {
    // text_time: pooled text embeds followed by one sinusoid per time id (SDXL base 6, SDXL refiner 5)
    const int ids_dim = d.projection_class_embeddings_input_dim - d.pooled_dim;
    CFGPP_REQUIRE(ids_dim > 0 && ids_dim % d.addition_time_embed_dim == 0,
                  "projection_class_embeddings_input_dim - pooled_dim must be a whole multiple of "
                  "addition_time_embed_dim");
    n_time_ids_ = ids_dim / d.addition_time_embed_dim;
    CFGPP_REQUIRE(n_time_ids_ >= 1 && n_time_ids_ <= 8, "the add-embedding must take 1..8 time ids");
  }
  CFGPP_REQUIRE(d.prediction_type == 0 || d.prediction_type == 1, "prediction_type must be 0 (epsilon) or 1 (v)");
  v_pred_ = d.prediction_type == 1;
  gemm_configure();
  attn_configure();
  CFGPP_CHECK_CUDA(cudaStreamCreateWithFlags(&capture_stream_, cudaStreamNonBlocking));
}

Unet::~Unet() {
  if (owner_) {  // the UNet's plan reads this handle's buffers: it must be built again
    owner_->cn_ = nullptr;
    owner_->prepared_ = false;
    owner_->graph_valid_ = false;
  }
  if (cn_) cn_->owner_ = nullptr;
  if (graph_exec_) cudaGraphExecDestroy(graph_exec_);
  if (graph_) cudaGraphDestroy(graph_);
  if (capture_stream_) cudaStreamDestroy(capture_stream_);
  if (noise_buf_) cudaFree(noise_buf_);
}

// ------------------------------------------------------------------------------------------------------------
// weights
// ------------------------------------------------------------------------------------------------------------
void Unet::load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                       cudaStream_t stream) {
  CFGPP_REQUIRE(!finalized_, "weights already finalized");
  weights_.load(key, data, shape, ndim, dtype, stream);
}

// ------------------------------------------------------------------------------------------------------------
// LoRA adapters
// ------------------------------------------------------------------------------------------------------------
void Unet::lora_add(int adapter, const std::string& key, const void* down, const void* up, int rank, float alpha,
                    int dtype, cudaStream_t stream) {
  CFGPP_REQUIRE(finalized_, "call cfgpp_finalize_weights first");
  weights_.lora_add(adapter, key, down, up, rank, alpha, dtype, stream);
}

void Unet::lora_set_scales(const float* scales, int n, cudaStream_t stream) {
  size_t bytes = 0;
  const std::set<std::string> touched = weights_.lora_apply(scales, n, stream, &bytes);
  prompt_stale_ = true;
  lora_bytes_moved_ = bytes + weights_.refresh(touched, stream);
}

void Unet::lora_clear(cudaStream_t stream) {
  size_t bytes = 0;
  const std::set<std::string> touched = weights_.lora_restore(stream, &bytes);
  prompt_stale_ = true;
  lora_bytes_moved_ = bytes + weights_.refresh(touched, stream);
  weights_.lora_free(stream);
}

void Unet::lora_stats(int* n_adapters, int* n_targets, size_t* backup_bytes, size_t* bytes_moved) const {
  if (n_adapters) *n_adapters = weights_.lora_adapters();
  if (n_targets) *n_targets = weights_.lora_targets();
  if (backup_bytes) *backup_bytes = weights_.lora_backup_bytes();
  if (bytes_moved) *bytes_moved = lora_bytes_moved_;
}

void Unet::require_fresh_prompt() const {
  CFGPP_REQUIRE(!prompt_stale_, "LoRA weights changed since cfgpp_set_prompt: call cfgpp_set_prompt again (the "
                                "cross-attention K/V and the add-embedding were computed from the previous weights)");
}

void Unet::finalize_weights(cudaStream_t stream) {
  CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));
  // structural validation: building a plan at a nominal size reads (and packs) every weight the plan touches
  finalized_ = true;
  try {
    // the smallest latent for which every level keeps a spatial extent (H, W >= 1 at the deepest level)
    const int s = 1 << (d_.num_levels - 1);
    if (is_cn_) {
      // the conditioning embedding's convolutions, zero-padded to whole 64-channel K blocks, and the zero convs
      auto pad64 = [](int c) { return (c + 63) / 64 * 64; };
      const int n = cn_desc_.num_embedding_levels;
      const int* ch = cn_desc_.embedding_channels;
      auto pack = [&](const std::string& name, int cin, int cout, int cout_p) {
        const std::string k = "controlnet_cond_embedding." + name;
        const WeightStore::Weight& w = weights_.raw(k + ".weight");
        CFGPP_REQUIRE(w.shape.size() == 4 && w.shape[0] == cout && w.shape[1] == cin && w.shape[2] == 3 &&
                          w.shape[3] == 3,
                      "unexpected shape of " + k + ".weight");
        weights_.plain(k + ".bias", cout);
        embed_convs_[name] = EmbedConv{weights_.packed_conv3x3(k + ".weight", pad64(cin), cout_p),
                                       weights_.packed_heads_rows({k + ".bias"}, 1, cout, cout_p), cout_p, pad64(cin)};
      };
      pack("conv_in", cn_desc_.conditioning_channels, ch[0], pad64(ch[0]));
      for (int i = 0; i + 1 < n; ++i) {
        pack("blocks." + std::to_string(2 * i), ch[i], ch[i], pad64(ch[i]));
        pack("blocks." + std::to_string(2 * i + 1), ch[i], ch[i + 1], pad64(ch[i + 1]));
      }
      pack("conv_out", ch[n - 1], d_.block_out_channels[0], d_.block_out_channels[0]);
      CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
      StreamKScope sk_scope(sk_.ws(), sk_.flags());
      build(1, std::max(8, s * 8), std::max(8, s * 8), nullptr);
      const std::vector<std::string> keys = zero_conv_keys();
      for (size_t k = 0; k < keys.size(); ++k) {
        const size_t C = res_[k].C;
        weights_.plain(keys[k] + ".weight", C * C);
        weights_.plain(keys[k] + ".bias", C);
      }
      CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
    } else {
      prepare(1, std::max(8, s * 8), std::max(8, s * 8));
    }
    prepared_ = false;
  } catch (...) {
    finalized_ = false;
    throw;
  }
}

// ------------------------------------------------------------------------------------------------------------
// workspace
// ------------------------------------------------------------------------------------------------------------
Unet::Scratch* Unet::scratch(const std::string& name, size_t numel_half) {
  auto& s = scratch_[name];
  if (!s) s.reset(new Scratch());
  if (s->p == nullptr) {
    s->need = std::max(s->need, numel_half);
  } else {
    CFGPP_REQUIRE(numel_half <= s->need, "scratch undersized: " + name);
  }
  return s.get();
}

// ------------------------------------------------------------------------------------------------------------
// plan building. The structure is walked twice by prepare(): a sizing pass (scratch buffers unallocated: only
// sizes are recorded, no ops are created) and the real pass.
// ------------------------------------------------------------------------------------------------------------
void Unet::add_step(const std::string& name, std::function<void(cudaStream_t)> fn, int launches) {
  if (sizing_) return;
  PlanStep s;
  s.name = name;
  s.fn = std::move(fn);
  s.launches = launches;
  cur_plan_->push_back(std::move(s));
}

void Unet::add_gemm(const std::string& name, const GemmOp& op, double algorithmic_flops) {
  PlanStep s;
  s.name = name;
  s.flops = algorithmic_flops >= 0 ? algorithmic_flops : op.flops();
  s.kind = op.p.conv ? 1 : 0;
  s.fn = [op](cudaStream_t st) { run_gemm_op(op, st); };
  cur_plan_->push_back(std::move(s));
}

void Unet::add_attn(const std::string& name, const AttnOp& op) {
  PlanStep s;
  s.name = name;
  s.flops = op.flops();
  s.kind = 2;
  s.fn = [op](cudaStream_t st) { run_attn_op(op, st); };
  cur_plan_->push_back(std::move(s));
}

Unet::Act Unet::build_resnet(const std::string& prefix, Act x1, const Act* x2, int Cout, int H, int W, int temb_off) {
  const int C1 = x1.C, C2 = x2 ? x2->C : 0, Cin = C1 + C2;
  const int HW = H * W;
  const size_t M = static_cast<size_t>(NB_) * HW;
  Scratch* s_norm = scratch("norm", M * std::max(Cin, Cout));
  Scratch* s_h1 = scratch("h1", M * Cout);
  Scratch* s_sc = (Cin != Cout) ? scratch("shortcut", M * Cout) : nullptr;
  if (sizing_) return Act{nullptr, Cout};
  __half* out = alloc_act(M * Cout);
  const __half* x2p = x2 ? x2->p : nullptr;
  const __half *g1 = weights_.plain(prefix + ".norm1.weight"), *b1 = weights_.plain(prefix + ".norm1.bias");
  const __half *g2 = weights_.plain(prefix + ".norm2.weight"), *b2 = weights_.plain(prefix + ".norm2.bias");
  const float eps = d_.norm_eps;
  float* partial = gn_partial_;
  const int NB = NB_;
  __half* normp = s_norm->p;
  __half* h1p = s_h1->p;
  const __half* x1p = x1.p;
  add_step(prefix + ".norm1+silu", [=](cudaStream_t st) {
    run_groupnorm(x1p, C1, x2p, C2, NB, HW, g1, b1, eps, true, partial, normp, st);
  }, 2);
  add_gemm(prefix + ".conv1", make_conv3x3_op(normp, NB_, H, W, Cin, weights_.packed_conv3x3(prefix + ".conv1.weight"), Cout,
                                              weights_.plain(prefix + ".conv1.bias"), temb_all_ + temb_off, temb_total_, HW, h1p));
  add_step(prefix + ".norm2+silu", [=](cudaStream_t st) {
    run_groupnorm(h1p, Cout, nullptr, 0, NB, HW, g2, b2, eps, true, partial, normp, st);
  }, 2);
  const __half* residual = x1p;
  if (Cin != Cout) {
    add_gemm(prefix + ".conv_shortcut",
             make_linear_op(x1p, C1, x2p, C2, C1, weights_.plain(prefix + ".conv_shortcut.weight"), static_cast<int>(M), Cout,
                            Cin, weights_.plain(prefix + ".conv_shortcut.bias"), nullptr, 0, 1, s_sc->p, Cout, false));
    residual = s_sc->p;
  }
  add_gemm(prefix + ".conv2", make_conv3x3_op(normp, NB_, H, W, Cout, weights_.packed_conv3x3(prefix + ".conv2.weight"), Cout,
                                              weights_.plain(prefix + ".conv2.bias"), residual, Cout, 1, out));
  return Act{out, Cout};
}

Unet::Act Unet::build_transformer(const std::string& prefix, Act x, int H, int W, int layers, int heads) {
  const int C = x.C;
  const int HW = H * W;
  const int Mi = NB_ * HW;
  const size_t M = static_cast<size_t>(Mi);
  const int D = d_.cross_attention_dim;
  CFGPP_REQUIRE(C % heads == 0 && C / heads <= 192,
                "attention supports head_dim <= 192 (got " + std::to_string(C / std::max(heads, 1)) + ") at " + prefix);
  const int hd = C / heads;
  const int hdp = attn_padded_head_dim(hd);  // heads are zero-padded to a multiple of 64 channels (SD v1.5: 40/80/160)
  const int Cp = heads * hdp;
  Scratch* s_norm = scratch("norm", M * C);
  Scratch* s_tok = scratch("tokens", M * C);
  Scratch* s_qkv = scratch("qkv", M * 3 * Cp);
  Scratch* s_attn = scratch("attn", M * Cp);
  Scratch* s_q = scratch("q", M * Cp);
  Scratch* s_ff = scratch("ff", M * 4 * C);
  Scratch* s_stats[3];
  for (int i = 0; i < 3; ++i)  // [16 N blocks][M] float2 partial row statistics (LayerNorm fold)
    s_stats[i] = scratch("lnstats" + std::to_string(i), static_cast<size_t>(32) * M * 2 * 2);
  if (sizing_) return Act{nullptr, C};
  __half* out = alloc_act(M * C);
  const int Mkv = NB_ * n_ctx_;
  const int NB = NB_;
  float* partial = gn_partial_;
  __half *normp = s_norm->p, *tok = s_tok->p, *qkv = s_qkv->p, *attn = s_attn->p, *qb = s_q->p, *ff = s_ff->p;
  // LayerNorm fold: the GEMMs that write the residual stream `tok` also emit per-row partial statistics, and the
  // GEMMs that read LN(tok) run on `tok` with gamma folded into the weight (no LayerNorm launches at all)
  float* stats[3];
  int parts[3] = {0, 0, 0};
  for (int i = 0; i < 3; ++i) stats[i] = reinterpret_cast<float*>(s_stats[i]->p);
  // a producer's N blocks must tile C exactly so that every column contributes to the row statistics
  auto producer = [&](const std::function<GemmOp(int)>& make, int slot) {
    GemmOp op = make(0);
    if (C % op.bn != 0) {
      for (int bn : {160, 128, 64})
        if (C % bn == 0) {
          op = make(bn);
          break;
        }
    }
    CFGPP_REQUIRE(C % op.bn == 0 && op.p.num_n_blocks <= 16, "LayerNorm fold: no tile width divides C");
    // two partial sums per N block: the epilogue splits a tile's columns between two warps per row
    op.p.stats_out = stats[slot];
    parts[slot] = 2 * op.p.num_n_blocks;
    return op;
  };
  auto consumer = [&](GemmOp op, const FoldedLN& f, int slot) {
    op.p.stats_in = stats[slot];
    op.p.ln_parts = parts[slot];
    op.p.ln_inv_c = 1.0f / static_cast<float>(C);
    op.p.ln_eps = 1e-5f;
    op.p.ln_s = f.s;
    op.p.ln_t = f.t;
    return op;
  };
  {
    const __half *g = weights_.plain(prefix + ".norm.weight"), *b = weights_.plain(prefix + ".norm.bias");
    const __half* xp = x.p;
    add_step(prefix + ".norm", [=](cudaStream_t st) {
      run_groupnorm(xp, C, nullptr, 0, NB, HW, g, b, 1e-6f, false, partial, normp, st);
    }, 2);
  }
  add_gemm(prefix + ".proj_in", producer([&](int bn) {
             return make_linear_op(normp, C, nullptr, 0, 0, weights_.plain(prefix + ".proj_in.weight"), Mi, C, C,
                                   weights_.plain(prefix + ".proj_in.bias"), nullptr, 0, 1, tok, C, false, bn);
           }, 0));
  for (int k = 0; k < layers; ++k) {
    const std::string b = prefix + ".transformer_blocks." + std::to_string(k);
    // --- self-attention ---
    __half* wqkv = weights_.packed_heads_rows({b + ".attn1.to_q.weight", b + ".attn1.to_k.weight", b + ".attn1.to_v.weight"},
                                     heads, hd, hdp);
    const FoldedLN f1 = weights_.folded_ln(b + ".attn1.qkv", {b + ".attn1.to_q.weight", b + ".attn1.to_k.weight", b + ".attn1.to_v.weight"}, wqkv, 3 * Cp, C, b + ".norm1", nullptr);
    add_gemm(b + ".attn1.to_qkv(+norm1)",
             consumer(make_linear_op(tok, C, nullptr, 0, 0, f1.w, Mi, 3 * Cp, C, nullptr, nullptr, 0, 1, qkv, 3 * Cp, false),
                      f1, 0),
             2.0 * Mi * 3.0 * C * C);
    add_attn(b + ".attn1.sdpa",
             make_attn_op(qkv, 3 * Cp, qkv + Cp, 3 * Cp, qkv + 2 * Cp, 3 * Cp, attn, Cp, NB_, heads, HW, HW, hd));
    add_gemm(b + ".attn1.to_out", producer([&](int bn) {
               return make_linear_op(attn, Cp, nullptr, 0, 0,
                                     weights_.packed_heads_cols(b + ".attn1.to_out.0.weight", heads, hd, hdp), Mi, C, Cp,
                                     weights_.plain(b + ".attn1.to_out.0.bias"), tok, C, 1, tok, C, false, bn);
             }, 1),
             2.0 * Mi * static_cast<double>(C) * C);
    // --- cross-attention (K/V projected once per prompt by the prompt plan) ---
    __half* wq2 = weights_.packed_heads_rows({b + ".attn2.to_q.weight"}, heads, hd, hdp);
    const FoldedLN f2 = weights_.folded_ln(b + ".attn2.q", {b + ".attn2.to_q.weight"}, wq2, Cp, C, b + ".norm2", nullptr);
    add_gemm(b + ".attn2.to_q(+norm2)",
             consumer(make_linear_op(tok, C, nullptr, 0, 0, f2.w, Mi, Cp, C, nullptr, nullptr, 0, 1, qb, Cp, false), f2, 1),
             2.0 * Mi * static_cast<double>(C) * C);
    __half* kv = alloc_act(static_cast<size_t>(Mkv) * 2 * Cp);
    {
      __half* wkv = weights_.packed_heads_rows({b + ".attn2.to_k.weight", b + ".attn2.to_v.weight"}, heads, hd, hdp);
      std::vector<PlanStep>* save = cur_plan_;
      cur_plan_ = &prompt_plan_;
      add_gemm(b + ".attn2.to_kv",
               make_linear_op(ctx_copy_, D, nullptr, 0, 0, wkv, Mkv, 2 * Cp, D, nullptr, nullptr, 0, 1, kv, 2 * Cp, false),
               2.0 * Mkv * 2.0 * C * D);
      cur_plan_ = save;
    }
    if (ip_ntok_ > 0 && !is_cn_) {  // IP-Adapter: the image tokens' K‖V once per image, attended to in the same kernel
      const int Mip = NB_ * ip_ntok_;
      __half* kv_ip = alloc_act(static_cast<size_t>(Mip) * 2 * Cp);
      const std::string pk = b + ".attn2.processor.to_k_ip.0.weight", pv = b + ".attn2.processor.to_v_ip.0.weight";
      weights_.plain(pk, static_cast<size_t>(C) * D);
      weights_.plain(pv, static_cast<size_t>(C) * D);
      __half* wkv = weights_.packed_heads_rows({pk, pv}, heads, hd, hdp);
      std::vector<PlanStep>* save = cur_plan_;
      cur_plan_ = &ip_plan_;
      add_gemm(b + ".attn2.to_kv_ip",
               make_linear_op(ip_tokens_, D, nullptr, 0, 0, wkv, Mip, 2 * Cp, D, nullptr, nullptr, 0, 1, kv_ip, 2 * Cp,
                              false),
               2.0 * Mip * 2.0 * C * D);
      cur_plan_ = save;
      add_attn(b + ".attn2.sdpa", make_attn_ip_op(qb, Cp, kv, 2 * Cp, kv + Cp, 2 * Cp, kv_ip, 2 * Cp, kv_ip + Cp, 2 * Cp,
                                                  ip_ntok_, &args_->ip_scale, attn, Cp, NB_, heads, HW, n_ctx_, hd));
    } else {
      add_attn(b + ".attn2.sdpa", make_attn_op(qb, Cp, kv, 2 * Cp, kv + Cp, 2 * Cp, attn, Cp, NB_, heads, HW, n_ctx_, hd));
    }
    add_gemm(b + ".attn2.to_out", producer([&](int bn) {
               return make_linear_op(attn, Cp, nullptr, 0, 0,
                                     weights_.packed_heads_cols(b + ".attn2.to_out.0.weight", heads, hd, hdp), Mi, C, Cp,
                                     weights_.plain(b + ".attn2.to_out.0.bias"), tok, C, 1, tok, C, false, bn);
             }, 2),
             2.0 * Mi * static_cast<double>(C) * C);
    // --- GEGLU feed-forward ---
    __half* wg = weights_.packed_geglu(b + ".ff.net.0.proj.weight", false);
    __half* bg = weights_.packed_geglu(b + ".ff.net.0.proj.bias", true);
    const FoldedLN f3 = weights_.folded_ln(b + ".ff.geglu", {b + ".ff.net.0.proj.weight"}, wg, 8 * C, C, b + ".norm3", bg);
    add_gemm(b + ".ff.geglu(+norm3)",
             consumer(make_linear_op(tok, C, nullptr, 0, 0, f3.w, Mi, 8 * C, C, nullptr, nullptr, 0, 1, ff, 4 * C, true), f3, 2));
    add_gemm(b + ".ff.out", producer([&](int bn) {
               return make_linear_op(ff, 4 * C, nullptr, 0, 0, weights_.plain(b + ".ff.net.2.weight"), Mi, C, 4 * C,
                                     weights_.plain(b + ".ff.net.2.bias"), tok, C, 1, tok, C, false, bn);
             }, 0));
  }
  add_gemm(prefix + ".proj_out", make_linear_op(tok, C, nullptr, 0, 0, weights_.plain(prefix + ".proj_out.weight"), Mi, C, C,
                                                weights_.plain(prefix + ".proj_out.bias"), x.p, C, 1, out, C, false));
  return Act{out, C};
}

Unet::Act Unet::build_downsample(const std::string& prefix, Act x, int H, int W) {
  const int C = x.C;
  const int Ho = H / 2, Wo = W / 2;
  const size_t Mo = static_cast<size_t>(NB_) * Ho * Wo;
  if (sizing_) return Act{nullptr, C};
  __half* out = alloc_act(Mo * C);
  // stride-2 conv as an implicit GEMM: the A tile of every tap comes through a tensor map with element strides 2
  add_gemm(prefix + ".conv", make_conv3x3_op(x.p, NB_, H, W, C, weights_.packed_conv3x3(prefix + ".conv.weight"), C,
                                             weights_.plain(prefix + ".conv.bias"), nullptr, 0, 1, out, 0, 2));
  return Act{out, C};
}

Unet::Act Unet::build_upsample(const std::string& prefix, Act x, int H, int W) {
  const int C = x.C;
  const size_t Mo = static_cast<size_t>(NB_) * 4 * H * W;
  Scratch* s_up = scratch("upsampled", Mo * C);
  if (sizing_) return Act{nullptr, C};
  __half* out = alloc_act(Mo * C);
  const int NB = NB_;
  const __half* xp = x.p;
  __half* up = s_up->p;
  add_step(prefix + ".nearest2x", [=](cudaStream_t st) { run_upsample2x(xp, up, NB, H, W, C, st); });
  add_gemm(prefix + ".conv", make_conv3x3_op(up, NB_, 2 * H, 2 * W, C, weights_.packed_conv3x3(prefix + ".conv.weight"), C,
                                             weights_.plain(prefix + ".conv.bias"), nullptr, 0, 1, out));
  return Act{out, C};
}

void Unet::prepare(int batch, int h_lat, int w_lat) {
  CFGPP_REQUIRE(!is_cn_, "a ControlNet handle is prepared through the UNet handle it is attached to");
  CFGPP_REQUIRE(finalized_, "call cfgpp_finalize_weights first");
  // validate BEFORE anything is freed: a rejected shape must leave the previous plan usable
  CFGPP_REQUIRE(batch >= 1 && 2 * batch <= 16, "batch must be 1..8 (UNet batch 2*batch <= 16)");
  {
    const int down = 1 << (d_.num_levels - 1);
    CFGPP_REQUIRE(h_lat >= down && w_lat >= down && h_lat % down == 0 && w_lat % down == 0,
                  "latent H, W must be multiples of 2^(num_levels-1)");
    // every level tiled-addressable (any size), or a latent of at least 64 x 64 whose other levels take the im2col
    // A tile
    bool tiled = true;
    for (int i = 0, h = h_lat, w = w_lat; i < d_.num_levels; ++i, h /= 2, w /= 2)
      tiled = tiled && conv3x3_geometry_supported(h, w);
    CFGPP_REQUIRE(tiled || latent_allows_im2col(h_lat, w_lat),
                  "latent " + std::to_string(h_lat) + "x" + std::to_string(w_lat) +
                      ": a latent whose levels are not all tiled-addressable (W % 128 == 0, or a power-of-two W <= 128 "
                      "with H a multiple of 128 / W) must be at least 64 x 64 (512 px images)");
  }
  CFGPP_CHECK_CUDA(cudaSetDevice(device_));
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
  StreamKScope sk_scope(sk_.ws(), sk_.flags());  // every GEMM op built below parks its stream-K partials in OUR workspace
  cn_image_ready_ = false;
  build(batch, h_lat, w_lat, nullptr);
  if (cn_) {
    // the ControlNet's ops are built under this handle's stream-K scope: they run on this handle's stream
    cn_->build(batch, h_lat, w_lat, args_);
    cn_->account();
    build_control_plan();
  }
  account();
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
  prepared_ = true;
}

void Unet::build(int batch, int h_lat, int w_lat, StepArgs* shared_args) {
  // from here on the old plan is gone: a throw below must not leave the handle looking prepared
  prepared_ = false;
  nsteps_ = 0;
  entries_.clear();
  v_ready_ = false;
  graph_valid_ = false;
  // drop the previous plan / workspace
  act_.clear();
  scratch_.clear();
  prologue_plan_.clear();
  body_plan_.clear();
  control_plan_.clear();
  up_plan_.clear();
  tail_plan_.clear();
  prompt_plan_.clear();
  ip_plan_.clear();
  ip_ready_ = false;
  t2i_feat_.clear();
  t2i_hw_.clear();
  t2i_ready_ = false;
  res_.clear();
  res_hw_.clear();
  B_ = batch; NB_ = 2 * batch; H_ = h_lat; W_ = w_lat;
  const int L = d_.num_levels;
  const int C0 = d_.block_out_channels[0];
  const int TE = time_embed_dim_;

  // resnet order (= temb offsets) is fixed by the structure walk below; compute it first
  temb_order_.clear();
  temb_total_ = 0;
  std::vector<std::string> temb_w_keys, temb_b_keys;
  auto reg_resnet = [&](const std::string& prefix, int Cout) {
    temb_order_.push_back({prefix, temb_total_});
    temb_total_ += Cout;
    temb_w_keys.push_back(prefix + ".time_emb_proj.weight");
    temb_b_keys.push_back(prefix + ".time_emb_proj.bias");
  };
  for (int i = 0; i < L; ++i)
    for (int j = 0; j < d_.layers_per_block; ++j)
      reg_resnet("down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), d_.block_out_channels[i]);
  reg_resnet("mid_block.resnets.0", d_.block_out_channels[L - 1]);
  reg_resnet("mid_block.resnets.1", d_.block_out_channels[L - 1]);
  for (int i = 0; i < (is_cn_ ? 0 : L); ++i)  // a ControlNet has no up path
    for (int j = 0; j < d_.layers_per_block + 1; ++j)
      reg_resnet("up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), d_.block_out_channels[L - 1 - i]);
  auto temb_off = [&](const std::string& prefix) {
    for (auto& p : temb_order_)
      if (p.first == prefix) return p.second;
    throw Error(-11, "internal: unknown resnet " + prefix);
  };

  for (int pass = 0; pass < 2; ++pass) {
    sizing_ = (pass == 0);
    if (!sizing_) {
      // allocate scratch + fixed buffers now that sizes are known
      for (auto& kv : scratch_) kv.second->p = alloc_act(kv.second->need);
      gn_partial_ = act_.alloc<float>(static_cast<size_t>(NB_) * 128 * 64);
      t_sin_ = alloc_act(C0);
      t_h1_ = alloc_act(TE);
      emb_ = alloc_act(static_cast<size_t>(NB_) * TE);
      semb_ = alloc_act(static_cast<size_t>(NB_) * TE);
      temb_all_ = alloc_act(static_cast<size_t>(NB_) * temb_total_);
      ctx_copy_ = alloc_act(static_cast<size_t>(NB_) * n_ctx_ * d_.cross_attention_dim);
      if (has_aug_) {
        add_in_ = alloc_act(static_cast<size_t>(NB_) * d_.projection_class_embeddings_input_dim);
        add_h1_ = alloc_act(static_cast<size_t>(NB_) * TE);
        aug_emb_ = alloc_act(static_cast<size_t>(NB_) * TE);
        pooled_copy_ = alloc_act(static_cast<size_t>(NB_) * d_.pooled_dim);
        time_ids_copy_ = act_.alloc<float>(static_cast<size_t>(NB_) * n_time_ids_);
      }
      args_ = shared_args ? shared_args : act_.alloc<StepArgs>(1);
      if (ip_ntok_ > 0 && !is_cn_) {
        if (ip_rs_.num_queries == 0) {  // the Resampler allocates its own buffers (build_ip_resampler)
          ip_embeds_ = alloc_act(static_cast<size_t>(NB_) * ip_embed_dim_);
          ip_proj_ = alloc_act(static_cast<size_t>(NB_) * ip_ntok_ * d_.cross_attention_dim);
        }
        ip_tokens_ = alloc_act(static_cast<size_t>(NB_) * ip_ntok_ * d_.cross_attention_dim);
      }
      if (!is_cn_) {  // the sampler state and tables: a ControlNet runs inside its UNet's step
        step_counter_ = act_.alloc<int>(1);
        step_table_ = act_.alloc<StepEntry>(1024);
        const size_t lat = static_cast<size_t>(B_) * 4 * H_ * W_;
        z_state_ = act_.alloc<float>(lat);
        aux_state_ = act_.alloc<float>(lat);
        z0t_state_ = act_.alloc<float>(lat);
        lambda_buf_ = act_.alloc<float>(B_);
        const StepArgs a{{}, noise_buf_, nullptr, ip_scale_};  // no guidance table: the schedule's scalar lambda
        CFGPP_CHECK_CUDA(cudaMemcpy(args_, &a, sizeof(a), cudaMemcpyHostToDevice));
        fwd_eps_uc_ = alloc_act(lat);
        fwd_eps_c_ = alloc_act(lat);
      } else {
        cond_ = alloc_act(static_cast<size_t>(B_) * H_ * W_ * C0);
      }
      temb_w_all_ = weights_.packed_cat_rows(temb_w_keys);
      temb_b_all_ = weights_.packed_cat_rows(temb_b_keys);
      conv_in_w_ = weights_.plain("conv_in.weight");
      conv_in_b_ = weights_.plain("conv_in.bias");
      if (!is_cn_) {
        conv_out_w_ = weights_.packed_conv3x3("conv_out.weight");
        conv_out_b_ = weights_.plain("conv_out.bias");
      }
    }

    // ---- prologue: timestep embedding -> per-resnet time_emb_proj (SURVEY A.2 step 1, ResnetBlock2D temb) ----
    cur_plan_ = &prologue_plan_;
    if (!sizing_) {
      const int NB = NB_;
      const __half *w1 = weights_.plain("time_embedding.linear_1.weight"), *b1 = weights_.plain("time_embedding.linear_1.bias");
      const __half *w2 = weights_.plain("time_embedding.linear_2.weight"), *b2 = weights_.plain("time_embedding.linear_2.bias");
      __half *t_sin = t_sin_, *t_h1 = t_h1_, *emb = emb_, *semb = semb_, *temb_all = temb_all_;
      const __half* aug = has_aug_ ? aug_emb_ : nullptr;
      const StepArgs* args = args_;
      const __half *wa = temb_w_all_, *ba = temb_b_all_;
      const int ttot = temb_total_;
      add_step("time_proj", [=](cudaStream_t st) { run_sincos_embed(&args->cur.s.t, 1, 1, C0, t_sin, C0, 0, st); });
      add_step("time_embedding.linear_1+silu", [=](cudaStream_t st) {
        run_small_linear(t_sin, C0, w1, b1, nullptr, 0, t_h1, TE, nullptr, 1, TE, C0, true, st);
      });
      add_step("time_embedding.linear_2(+aug_emb)", [=](cudaStream_t st) {
        run_small_linear(t_h1, 0, w2, b2, aug, TE, emb, TE, semb, NB, TE, TE, false, st);
      });
      add_step("resnets.time_emb_proj", [=](cudaStream_t st) {
        run_small_linear(semb, TE, wa, ba, nullptr, 0, temb_all, ttot, nullptr, NB, ttot, TE, false, st);
      });
    }

    // ---- prompt plan: add-embedding (SDXL text_time) ----
    cur_plan_ = &prompt_plan_;
    if (!sizing_ && has_aug_) {
      const int NB = NB_;
      const int ATE = d_.addition_time_embed_dim, PD = d_.pooled_dim, AIN = d_.projection_class_embeddings_input_dim;
      const int NT = n_time_ids_;
      const __half *w1 = weights_.plain("add_embedding.linear_1.weight"), *b1 = weights_.plain("add_embedding.linear_1.bias");
      const __half *w2 = weights_.plain("add_embedding.linear_2.weight"), *b2 = weights_.plain("add_embedding.linear_2.bias");
      __half *add_in = add_in_, *add_h1 = add_h1_, *aug = aug_emb_, *pooled = pooled_copy_;
      float* tids = time_ids_copy_;
      add_step("add_embedding.assemble", [=](cudaStream_t st) {
        run_copy_rows(pooled, NB, PD, add_in, AIN, 0, NB, st);
        for (int j = 0; j < NT; ++j) run_sincos_embed(tids + j, NT, NB, ATE, add_in, AIN, PD + j * ATE, st);
      }, 1 + NT);
      add_step("add_embedding.linear_1+silu", [=](cudaStream_t st) {
        run_small_linear(add_in, AIN, w1, b1, nullptr, 0, add_h1, TE, nullptr, NB, TE, AIN, true, st);
      });
      add_step("add_embedding.linear_2", [=](cudaStream_t st) {
        run_small_linear(add_h1, TE, w2, b2, nullptr, 0, aug, TE, nullptr, NB, TE, TE, false, st);
      });
    }

    // ---- IP-Adapter image projection (diffusers ImageProjection): LayerNorm(D) of the rows of Linear(E -> ntok * D) ----
    cur_plan_ = &ip_plan_;
    if (!sizing_ && ip_ntok_ > 0 && !is_cn_ && ip_rs_.num_queries > 0) {
      build_ip_resampler();  // IP-Adapter Plus
    } else if (!sizing_ && ip_ntok_ > 0 && !is_cn_) {
      const int NB = NB_, D = d_.cross_attention_dim, E = ip_embed_dim_, T = ip_ntok_;
      add_gemm("image_proj.proj",
               make_linear_op(ip_embeds_, E, nullptr, 0, 0, weights_.plain("image_proj.proj.weight", size_t(T) * D * E),
                              NB, T * D, E, weights_.plain("image_proj.proj.bias", size_t(T) * D), nullptr, 0, 1,
                              ip_proj_, T * D, false));
      const __half *g = weights_.plain("image_proj.norm.weight", D), *bt = weights_.plain("image_proj.norm.bias", D);
      __half *in = ip_proj_, *out = ip_tokens_;
      add_step("image_proj.norm", [=](cudaStream_t st) { run_layernorm(in, NB * T, D, g, bt, 1e-5f, out, st); });
    }

    // ---- body (SURVEY A.2 steps 2-6) ----
    cur_plan_ = &body_plan_;
    const int HW0 = H_ * W_;
    const Act h0{sizing_ ? nullptr : alloc_act(static_cast<size_t>(NB_) * HW0 * C0), C0};
    Act h = h0;
    int H = H_, W = W_;
    std::vector<Act> skips{h};
    for (int i = 0; i < L; ++i) {
      const std::string blk = "down_blocks." + std::to_string(i);
      const int Cout = d_.block_out_channels[i];
      for (int j = 0; j < d_.layers_per_block; ++j) {
        const std::string rp = blk + ".resnets." + std::to_string(j);
        h = build_resnet(rp, h, nullptr, Cout, H, W, temb_off(rp));
        if (d_.down_has_attn[i]) {
          h = build_transformer(blk + ".attentions." + std::to_string(j), h, H, W, d_.transformer_layers[i],
                                d_.num_heads[i]);
          if (j == d_.layers_per_block - 1) add_t2i_feature(h, H, W);  // before the downsampler
        }
        skips.push_back(h);
      }
      if (i != L - 1) {
        h = build_downsample(blk + ".downsamplers.0", h, H, W);
        H /= 2; W /= 2;
        skips.push_back(h);
      }
      if (!d_.down_has_attn[i]) add_t2i_feature(h, H, W);  // DownBlock2D: its output, in place under the skip
    }
    {
      const int Cm = d_.block_out_channels[L - 1];
      h = build_resnet("mid_block.resnets.0", h, nullptr, Cm, H, W, temb_off("mid_block.resnets.0"));
      h = build_transformer("mid_block.attentions.0", h, H, W, d_.transformer_layers[L - 1], d_.num_heads[L - 1]);
      h = build_resnet("mid_block.resnets.1", h, nullptr, Cm, H, W, temb_off("mid_block.resnets.1"));
      add_t2i_feature(h, H, W);  // the feature left over (t2i_n_ = L + 1), of the last down placement's shape
      CFGPP_REQUIRE(sizing_ || is_cn_ || static_cast<int>(t2i_feat_.size()) == t2i_n_,
                    "internal: T2I-Adapter placements differ from the attached feature count");
    }
    if (!sizing_) {
      conv_in_out_ = h0.p;
      res_ = skips;
      res_.push_back(h);
      for (int i = 0, hh = H_, ww = W_; i < L; ++i, hh /= 2, ww /= 2)
        for (int j = 0; j < d_.layers_per_block + (i == 0 ? 1 : 0) + (i != L - 1 ? 1 : 0); ++j)
          res_hw_.push_back(j == d_.layers_per_block + (i == 0 ? 1 : 0) && i != L - 1 ? (hh / 2) * (ww / 2) : hh * ww);
      res_hw_.push_back(H * W);
    }
    if (is_cn_) continue;  // a ControlNet's plan ends with its mid block
    cur_plan_ = &up_plan_;
    for (int i = 0; i < L; ++i) {
      const std::string blk = "up_blocks." + std::to_string(i);
      const int rev = L - 1 - i;
      const int Cout = d_.block_out_channels[rev];
      for (int j = 0; j < d_.layers_per_block + 1; ++j) {
        Act skip = skips.back();
        skips.pop_back();
        const std::string rp = blk + ".resnets." + std::to_string(j);
        h = build_resnet(rp, h, &skip, Cout, H, W, temb_off(rp));
        if (d_.up_has_attn[i])
          h = build_transformer(blk + ".attentions." + std::to_string(j), h, H, W, d_.transformer_layers[rev],
                                d_.num_heads[rev]);
      }
      if (i != L - 1) {
        h = build_upsample(blk + ".upsamplers.0", h, H, W);
        H *= 2; W *= 2;
      }
    }
    CFGPP_REQUIRE(skips.empty() && H == H_ && W == W_, "internal: skip stack mismatch");
    // ---- tail: conv_norm_out + SiLU on the last up block's output feeds the fused conv_out / CFG++ step kernel ----
    cur_plan_ = &tail_plan_;
    Scratch* s_norm = scratch("tail.norm", static_cast<size_t>(NB_) * HW0 * C0);
    if (!sizing_) {
      const __half *g = weights_.plain("conv_norm_out.weight"), *b = weights_.plain("conv_norm_out.bias");
      const int NB = NB_, HW = HW0;
      const float eps = d_.norm_eps;
      float* partial = gn_partial_;
      __half* normp = s_norm->p;
      const __half* hp = h.p;
      add_step("conv_norm_out+silu", [=](cudaStream_t st) {
        run_groupnorm(hp, C0, nullptr, 0, NB, HW, g, b, eps, true, partial, normp, st);
      }, 2);
      final_norm_ = Act{normp, C0};
    }
  }
  if (is_cn_ && shared_args) prepared_ = true;  // built for its UNet: set_prompt may run
}

void Unet::account() {
  // FLOP / launch accounting (the reference executes the K/V projections every step: count them per forward)
  const int C0 = d_.block_out_channels[0];
  const int TE = time_embed_dim_;
  forward_flops_ = 0.0;
  launches_per_step_ = is_cn_ ? 1 : 3;  // (select_step +) conv_in (+ conv_out_step)
  for (auto* pl : {&body_plan_, &control_plan_, &up_plan_, &tail_plan_})
    for (auto& s : *pl) { forward_flops_ += s.flops; launches_per_step_ += s.launches; }
  for (auto& s : prologue_plan_) launches_per_step_ += s.launches;
  prompt_flops_ = 0.0;
  prompt_launches_ = 0;
  for (auto* pl : {&prompt_plan_, &ip_plan_})
    for (auto& s : *pl) { prompt_flops_ += s.flops; prompt_launches_ += s.launches; }
  forward_flops_ += prompt_flops_;
  const double px = static_cast<double>(NB_) * H_ * W_;
  forward_flops_ += 2.0 * px * (36.0 * C0 + (is_cn_ ? 0.0 : 36.0 * C0));  // conv_in + conv_out
  forward_flops_ += 2.0 * NB_ * (static_cast<double>(C0) * TE + static_cast<double>(TE) * TE +
                                 static_cast<double>(temb_total_) * TE);
  if (has_aug_) {  // the add-embedding MLP runs in the prompt plan
    const double f = 2.0 * NB_ * (static_cast<double>(d_.projection_class_embeddings_input_dim) * TE +
                                  static_cast<double>(TE) * TE);
    forward_flops_ += f;
    prompt_flops_ += f;
  }
  if (cn_) {
    forward_flops_ += cn_->forward_flops_;
    launches_per_step_ += cn_->launches_per_step_;
    prompt_flops_ += cn_->prompt_flops_;
    prompt_launches_ += cn_->prompt_launches_;
  }
}

std::vector<std::string> Unet::zero_conv_keys() const {
  std::vector<std::string> keys;
  for (size_t k = 0; k + 1 < res_.size(); ++k) keys.push_back("controlnet_down_blocks." + std::to_string(k));
  keys.push_back("controlnet_mid_block");
  return keys;
}

void Unet::build_control_plan() {
  // zero conv k: a 1x1 convolution of the ControlNet's k-th residual, scaled and added in place into the UNet's k-th
  // skip tensor (the last: the mid-block output). The UNet's down path and mid block have consumed these tensors by
  // the time this plan runs, so only the up path sees the sums.
  CFGPP_REQUIRE(cn_->res_.size() == res_.size(), "internal: ControlNet residual count differs from the UNet's");
  cur_plan_ = &control_plan_;
  const std::vector<std::string> keys = cn_->zero_conv_keys();
  for (size_t k = 0; k < res_.size(); ++k) {
    const int C = res_[k].C;
    CFGPP_REQUIRE(cn_->res_[k].C == C && cn_->res_hw_[k] == res_hw_[k], "internal: ControlNet residual shape mismatch");
    const int M = NB_ * res_hw_[k];
    GemmOp op = make_linear_op(cn_->res_[k].p, C, nullptr, 0, 0, cn_->weights_.plain(keys[k] + ".weight", size_t(C) * C),
                               M, C, C, cn_->weights_.plain(keys[k] + ".bias", C), res_[k].p, C, 1, res_[k].p, C, false);
    op.p.res_scale = &args_->cur.control_scale;
    add_gemm(keys[k], op);
  }
}

void Unet::add_t2i_feature(Act h, int H, int W) {
  // in place on the block's output: its producer (proj_out, the downsample conv or a resnet's conv2) computes no row
  // statistics, and every later reader (the next block's GroupNorm, the downsampler, the skip) runs after the add
  if (sizing_ || is_cn_ || static_cast<int>(t2i_feat_.size()) >= t2i_n_) return;
  const int k = static_cast<int>(t2i_feat_.size());
  const size_t per_image = static_cast<size_t>(H) * W * h.C;
  __half* feat = alloc_act(static_cast<size_t>(B_) * per_image);
  t2i_feat_.push_back(Act{feat, h.C});
  t2i_hw_.push_back(H * W);
  const int NB = NB_, B = B_;
  __half* hp = h.p;
  const int* on = &args_->cur.t2i_on;
  add_step("t2i_adapter.add" + std::to_string(k),
           [=](cudaStream_t st) { run_t2i_add(hp, feat, NB, B, per_image, on, st); });
}

void Unet::run_plan(const std::vector<PlanStep>& plan, cudaStream_t stream) {
  for (const auto& s : plan) s.fn(stream);
}

// Body of the forward: conv_in output .. conv_norm_out, on the caller's stream.
void Unet::run_body(cudaStream_t stream) {
  if (cn_) run_plan(cn_->body_plan_, stream);
  run_plan(body_plan_, stream);
  run_plan(control_plan_, stream);
  run_plan(up_plan_, stream);
  run_plan(tail_plan_, stream);
}

// Prologue: the timestep embeddings; then conv_in (and the ControlNet's conv_in + conditioning embedding) on z.
void Unet::run_inputs(const void* z, int z_is_half, cudaStream_t stream) {
  run_plan(prologue_plan_, stream);
  if (cn_) run_plan(cn_->prologue_plan_, stream);
  const int C0 = d_.block_out_channels[0];
  const float* in_scale = &args_->cur.s.in_scale;
  run_conv_in(z, z_is_half, in_scale, conv_in_w_, conv_in_b_, conv_in_out_, B_, H_, W_, C0, 2, stream);
  if (cn_)
    run_conv_in(z, z_is_half, in_scale, cn_->conv_in_w_, cn_->conv_in_b_, cn_->conv_in_out_, B_, H_, W_, C0, 2, stream,
                cn_->cond_);
}

void Unet::require_ip_ready() const {
  CFGPP_REQUIRE(ip_ntok_ == 0 || ip_ready_, std::string("an IP-Adapter is attached: call ") +
                                                (ip_rs_.num_queries ? "cfgpp_set_ip_image_hidden_states"
                                                                    : "cfgpp_set_ip_image_embeds") +
                                                " for the prepared plan and the loaded adapter");
}

void Unet::require_control_ready() const {
  CFGPP_REQUIRE(!cn_ || cn_image_ready_, "a ControlNet is attached: call cfgpp_set_control_image for the prepared shape");
}

void Unet::require_t2i_ready() const {
  CFGPP_REQUIRE(t2i_n_ == 0 || t2i_ready_,
                "T2I-Adapter features are attached: call cfgpp_set_t2i_features for the prepared plan");
}

void Unet::upload_entries(cudaStream_t stream) {
  // pageable source: staged before the call returns; the stream orders it after a replay still reading the table
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(step_table_, entries_.data(), sizeof(StepEntry) * nsteps_, cudaMemcpyHostToDevice,
                                   stream));
}

void Unet::stage_entry(float t, float in_scale, cudaStream_t stream) {
  StepEntry e{};
  e.s.t = t;
  e.s.in_scale = in_scale;
  e.control_scale = cn_scale_;
  e.t2i_on = t2i_on_;
  // cudaMemcpyAsync from pageable memory stages the 64 bytes before returning: `e` may go out of scope
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(&args_->cur, &e, sizeof(e), cudaMemcpyHostToDevice, stream));
}

// ------------------------------------------------------------------------------------------------------------
// conditioning
// ------------------------------------------------------------------------------------------------------------
void Unet::set_prompt(const __half* ctx, int n_ctx, const __half* pooled, const float* time_ids, int add_rows,
                      cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(n_ctx == n_ctx_, "context length differs from the prepared plan (77)");
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(ctx_copy_, ctx, static_cast<size_t>(NB_) * n_ctx_ * d_.cross_attention_dim * 2,
                                   cudaMemcpyDeviceToDevice, stream));
  if (has_aug_) {
    CFGPP_REQUIRE(pooled && time_ids, "SDXL add-embedding needs pooled text embeds and time ids");
    CFGPP_REQUIRE(add_rows == NB_ || add_rows == B_, "add_rows must be batch or 2*batch");
    // broadcast rows r -> r % add_rows (the un-duplicated case of latent_sdxl.py:249-252)
    for (int r0 = 0; r0 < NB_; r0 += add_rows) {
      CFGPP_CHECK_CUDA(cudaMemcpyAsync(pooled_copy_ + static_cast<size_t>(r0) * d_.pooled_dim, pooled,
                                       static_cast<size_t>(add_rows) * d_.pooled_dim * 2, cudaMemcpyDeviceToDevice,
                                       stream));
      CFGPP_CHECK_CUDA(cudaMemcpyAsync(time_ids_copy_ + static_cast<size_t>(r0) * n_time_ids_, time_ids,
                                       static_cast<size_t>(add_rows) * n_time_ids_ * sizeof(float),
                                       cudaMemcpyDeviceToDevice, stream));
    }
  }
  run_plan(prompt_plan_, stream);
  if (cn_) cn_->set_prompt(ctx, n_ctx, pooled, time_ids, add_rows, stream);
  prompt_stale_ = false;
}

// ------------------------------------------------------------------------------------------------------------
// un-fused forward == predict_noise
// ------------------------------------------------------------------------------------------------------------
void Unet::unet_forward(const void* z, int z_dtype, float t, float in_scale, __half* eps_uc, __half* eps_c,
                        cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  require_fresh_prompt();
  require_control_ready();
  require_ip_ready();
  require_t2i_ready();
  stage_entry(t, in_scale, stream);
  run_inputs(z, z_dtype == CFGPP_F16 ? 1 : 0, stream);
  run_body(stream);
  run_conv_out_step(final_norm_.p, conv_out_w_, conv_out_b_, B_, H_, W_, final_norm_.C, STEP_NONE, nullptr, nullptr,
                    nullptr, nullptr, eps_uc, eps_c, stream);
}

std::vector<Unet::ProfEntry> Unet::profile_forward(const void* z, int z_dtype, float t, float in_scale,
                                                   cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  std::vector<ProfEntry> out;
  std::vector<cudaEvent_t> evs;
  auto mark = [&]() {
    cudaEvent_t e;
    CFGPP_CHECK_CUDA(cudaEventCreate(&e));
    CFGPP_CHECK_CUDA(cudaEventRecord(e, stream));
    evs.push_back(e);
  };
  require_control_ready();
  require_ip_ready();
  require_t2i_ready();
  stage_entry(t, in_scale, stream);
  mark();
  auto run = [&](const std::vector<PlanStep>& plan, const std::string& prefix) {
    for (const auto& st : plan) {
      st.fn(stream);
      mark();
      out.push_back({prefix + st.name, st.kind, st.flops, 0.f});
    }
  };
  const std::string cnp = "controlnet:";
  run(prologue_plan_, "");
  if (cn_) run(cn_->prologue_plan_, cnp);
  const int C0 = d_.block_out_channels[0];
  const double conv_in_flops = 2.0 * NB_ * H_ * W_ * 36.0 * C0;
  run_conv_in(z, z_dtype == CFGPP_F16 ? 1 : 0, &args_->cur.s.in_scale, conv_in_w_, conv_in_b_, conv_in_out_, B_, H_,
              W_, C0, 2, stream);
  mark();
  out.push_back({"conv_in", 3, conv_in_flops, 0.f});
  if (cn_) {
    run_conv_in(z, z_dtype == CFGPP_F16 ? 1 : 0, &args_->cur.s.in_scale, cn_->conv_in_w_, cn_->conv_in_b_,
                cn_->conv_in_out_, B_, H_, W_, C0, 2, stream, cn_->cond_);
    mark();
    out.push_back({cnp + "conv_in(+cond)", 3, conv_in_flops, 0.f});
    run(cn_->body_plan_, cnp);
  }
  for (auto* pl : {&body_plan_, &control_plan_, &up_plan_, &tail_plan_}) run(*pl, "");
  run_conv_out_step(final_norm_.p, conv_out_w_, conv_out_b_, B_, H_, W_, final_norm_.C, STEP_NONE, nullptr, nullptr,
                    nullptr, nullptr, fwd_eps_uc_, fwd_eps_c_, stream);
  mark();
  out.push_back({"conv_out+step", 3, 2.0 * NB_ * H_ * W_ * 36.0 * d_.block_out_channels[0], 0.f});
  CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));
  for (size_t i = 0; i < out.size(); ++i) CFGPP_CHECK_CUDA(cudaEventElapsedTime(&out[i].ms, evs[i], evs[i + 1]));
  for (auto e : evs) cudaEventDestroy(e);
  return out;
}

// ------------------------------------------------------------------------------------------------------------
// fused trajectory
// ------------------------------------------------------------------------------------------------------------
void Unet::set_schedule(int method, int state_dtype, const cfgpp_step_state* steps, int nsteps, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(method >= CFGPP_STEP_DDIM_CFGPP && method <= CFGPP_STEP_DDIM_CFG, "unknown method");
  CFGPP_REQUIRE(nsteps >= 1 && nsteps <= 1024, "nsteps must be 1..1024");
  static_assert(sizeof(cfgpp_step_state) == sizeof(StepState), "ABI struct mismatch");
  static_assert(sizeof(cfgpp_step_coef) == sizeof(StepCoef), "ABI struct mismatch");
  if (method != method_ || state_dtype != state_dtype_) graph_valid_ = false;
  method_ = method;
  state_dtype_ = state_dtype;
  nsteps_ = nsteps;
  // v coefficients and per-entry conditioning scales belong to the schedule they were set for
  entries_.assign(nsteps, StepEntry{});
  for (int i = 0; i < nsteps; ++i) {
    std::memcpy(&entries_[i].s, &steps[i], sizeof(StepState));
    entries_[i].control_scale = cn_scale_;
    entries_[i].t2i_on = t2i_on_;
  }
  v_ready_ = false;
  upload_entries(stream);
}

void Unet::set_v_coefs(const float* ab, int nsteps, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_ && nsteps_ > 0, "call cfgpp_set_schedule first");
  CFGPP_REQUIRE(v_pred_, "v coefficients belong to a prediction_type = 1 model");
  CFGPP_REQUIRE(ab != nullptr && nsteps == nsteps_, "one (a, b) pair per schedule entry");
  for (int i = 0; i < nsteps; ++i) entries_[i].v_ab = make_float2(ab[2 * i], ab[2 * i + 1]);
  upload_entries(stream);
  v_ready_ = true;
}

void Unet::set_state(const void* z, int z_dtype, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(z_dtype == state_dtype_, "state dtype differs from the schedule's state dtype");
  const size_t lat = static_cast<size_t>(B_) * 4 * H_ * W_;
  const size_t es = (state_dtype_ == CFGPP_F16) ? 2 : 4;
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(z_state_, z, lat * es, cudaMemcpyDeviceToDevice, stream));
}

void Unet::set_noise(const __half* noise, int slots, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(noise != nullptr && slots >= 1 && slots <= 1024, "noise table: 1..1024 slots");
  const size_t n = static_cast<size_t>(slots) * B_ * 4 * H_ * W_;
  if (n > noise_cap_) {
    CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));  // a replay in flight may still read the old table
    if (noise_buf_) cudaFree(noise_buf_);
    noise_buf_ = nullptr;
    noise_cap_ = 0;
    CFGPP_CHECK_CUDA(cudaMalloc(&noise_buf_, n * sizeof(__half)));
    noise_cap_ = n;
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(&args_->noise, &noise_buf_, sizeof(__half*), cudaMemcpyHostToDevice, stream));
    CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));  // &noise_buf_ is host memory of this object: do not let it race
  }
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(noise_buf_, noise, n * sizeof(__half), cudaMemcpyDeviceToDevice, stream));
}

void Unet::set_guidance(const float* lambda, int n, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(n == 0 || (lambda != nullptr && n == B_), "guidance table: n = 0 (clear) or one entry per image");
  // both copies come from pageable host memory, which cudaMemcpyAsync stages before it returns; the stream orders
  // them after any replay still reading the previous table
  if (n > 0)
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(lambda_buf_, lambda, static_cast<size_t>(n) * sizeof(float),
                                     cudaMemcpyHostToDevice, stream));
  const float* table = n > 0 ? lambda_buf_ : nullptr;
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(&args_->lambda, &table, sizeof(table), cudaMemcpyHostToDevice, stream));
}

void Unet::ensure_graph(cudaStream_t stream) {
  if (graph_valid_) return;
  if (graph_exec_) { cudaGraphExecDestroy(graph_exec_); graph_exec_ = nullptr; }
  if (graph_) { cudaGraphDestroy(graph_); graph_ = nullptr; }
  const int mode = method_ | (state_dtype_ == CFGPP_F16 ? 0x100 : 0);
  CFGPP_CHECK_CUDA(cudaStreamBeginCapture(capture_stream_, cudaStreamCaptureModeRelaxed));
  try {
    run_select_step(step_table_, step_counter_, args_, capture_stream_);
    run_inputs(z_state_, state_dtype_ == CFGPP_F16 ? 1 : 0, capture_stream_);
    run_body(capture_stream_);
    run_conv_out_step(final_norm_.p, conv_out_w_, conv_out_b_, B_, H_, W_, final_norm_.C, mode, args_, z_state_,
                      aux_state_, z0t_state_, nullptr, nullptr, capture_stream_, v_pred_);
  } catch (...) {
    cudaGraph_t g = nullptr;
    cudaStreamEndCapture(capture_stream_, &g);
    if (g) cudaGraphDestroy(g);
    throw;
  }
  CFGPP_CHECK_CUDA(cudaStreamEndCapture(capture_stream_, &graph_));
  CFGPP_CHECK_CUDA(cudaGraphInstantiate(&graph_exec_, graph_, 0));
  graph_valid_ = true;
  ++graph_captures_;
}

void Unet::run_steps(int first_step, int nsteps, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_ && nsteps_ > 0, "call cfgpp_set_schedule first");
  CFGPP_REQUIRE(first_step >= 0 && first_step + nsteps <= nsteps_, "step range outside the schedule");
  CFGPP_REQUIRE(!v_pred_ || v_ready_, "a v-prediction model needs cfgpp_set_v_coefs for this schedule");
  require_fresh_prompt();
  require_control_ready();
  require_ip_ready();
  require_t2i_ready();
  ensure_graph(stream);
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(step_counter_, &first_step, sizeof(int), cudaMemcpyHostToDevice, stream));
  for (int i = 0; i < nsteps; ++i) CFGPP_CHECK_CUDA(cudaGraphLaunch(graph_exec_, stream));
}

void Unet::get_state(int which, void* out, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  const size_t lat = static_cast<size_t>(B_) * 4 * H_ * W_;
  const size_t es = (state_dtype_ == CFGPP_F16) ? 2 : 4;
  const void* src = which == 0 ? z_state_ : (which == 1 ? z0t_state_ : aux_state_);
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(out, src, lat * es, cudaMemcpyDeviceToDevice, stream));
}

void Unet::apply_step(int step, const __half* eps_uc, const __half* eps_c, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_ && step >= 0 && step < nsteps_, "step outside the schedule");
  const int mode = method_ | (state_dtype_ == CFGPP_F16 ? 0x100 : 0);
  const int n = B_ * 4 * H_ * W_;
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(&args_->cur, step_table_ + step, sizeof(StepEntry), cudaMemcpyDeviceToDevice,
                                   stream));
  run_step_only(eps_uc, eps_c, n, mode, args_, z_state_, aux_state_, z0t_state_, 4 * H_ * W_, stream);
}

// ------------------------------------------------------------------------------------------------------------
// ControlNet
// ------------------------------------------------------------------------------------------------------------
void Unet::attach_controlnet(Unet* cn) {
  CFGPP_REQUIRE(!is_cn_, "a ControlNet attaches to a UNet handle, not to another ControlNet");
  if (cn) {
    CFGPP_REQUIRE(cn->is_cn_, "the handle to attach is not a ControlNet handle (cfgpp_controlnet_create)");
    CFGPP_REQUIRE(cn->finalized_, "call cfgpp_finalize_weights on the ControlNet first");
    CFGPP_REQUIRE(cn->device_ == device_, "the ControlNet lives on another device");
    CFGPP_REQUIRE(cn->owner_ == nullptr || cn->owner_ == this, "the ControlNet is attached to another UNet handle");
    const cfgpp_model_desc& c = cn->d_;
    auto same = [](bool ok, const char* field) {
      CFGPP_REQUIRE(ok, std::string("ControlNet ") + field + " differs from the UNet's");
    };
    same(c.num_levels == d_.num_levels, "num_levels");
    for (int i = 0; i < d_.num_levels; ++i) same(c.block_out_channels[i] == d_.block_out_channels[i], "block_out_channels");
    same(c.layers_per_block == d_.layers_per_block, "layers_per_block");
    same(c.cross_attention_dim == d_.cross_attention_dim, "cross_attention_dim");
    same(c.addition_time_embed_dim == d_.addition_time_embed_dim, "addition_time_embed_dim");
    if (has_aug_) {
      same(c.projection_class_embeddings_input_dim == d_.projection_class_embeddings_input_dim,
           "projection_class_embeddings_input_dim");
      same(c.pooled_dim == d_.pooled_dim, "pooled_dim");
    }
  }
  if (cn_ && cn_ != cn) cn_->owner_ = nullptr;
  cn_ = cn;
  if (cn) cn->owner_ = this;
  // the plan changes shape: the next cfgpp_prepare builds it
  prepared_ = false;
  graph_valid_ = false;
  nsteps_ = 0;
  cn_image_ready_ = false;
}

void Unet::set_control_image(const void* image, int dtype, cudaStream_t stream) {
  CFGPP_REQUIRE(cn_ != nullptr, "no ControlNet attached");
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(image != nullptr && (dtype == CFGPP_F16 || dtype == CFGPP_F32), "control image: fp16 or fp32 tensor");
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  cn_->cond_embed(image, dtype == CFGPP_F16, B_, 8 * H_, 8 * W_, cn_->cond_, stream);
  cn_image_ready_ = true;
}

void Unet::set_control_scale(float scale, cudaStream_t stream) {
  CFGPP_REQUIRE(!is_cn_, "the conditioning scale is set on the UNet handle");
  cn_scale_ = scale;
  for (StepEntry& e : entries_) e.control_scale = scale;
  if (cn_ && prepared_) upload_entries(stream);
}

void Unet::set_control_scales(const float* scales, int n, cudaStream_t stream) {
  CFGPP_REQUIRE(cn_ != nullptr && prepared_, "attach a ControlNet and call cfgpp_prepare first");
  CFGPP_REQUIRE(nsteps_ > 0 && scales != nullptr && n == nsteps_, "one conditioning scale per schedule entry");
  for (int i = 0; i < n; ++i) entries_[i].control_scale = scales[i];
  upload_entries(stream);
}

// ------------------------------------------------------------------------------------------------------------
// IP-Adapter
// ------------------------------------------------------------------------------------------------------------
void Unet::ip_load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                          cudaStream_t stream) {
  CFGPP_REQUIRE(!is_cn_, "an IP-Adapter loads into a UNet handle, not a ControlNet");
  CFGPP_REQUIRE(finalized_, "call cfgpp_finalize_weights first");
  const bool proj = key.rfind("image_proj.", 0) == 0;
  const bool kv = key.find(".attn2.processor.to_k_ip.0.weight") != std::string::npos ||
                  key.find(".attn2.processor.to_v_ip.0.weight") != std::string::npos;
  CFGPP_REQUIRE(proj || kv, "not an IP-Adapter weight key: " + key);
  if (kv) {  // [C, D] like the block's own to_k
    const std::string base = key.substr(0, key.find(".attn2.processor."));
    CFGPP_REQUIRE(weights_.has(base + ".attn2.to_k.weight"), "no cross-attention at " + base + " for " + key);
    const std::vector<int64_t>& want = weights_.raw(base + ".attn2.to_k.weight").shape;
    CFGPP_REQUIRE(static_cast<size_t>(ndim) == want.size() && std::equal(want.begin(), want.end(), shape),
                  "shape of " + key + " differs from the block's to_k");
  }
  // a key loaded again gets a new buffer: the plan, which holds raw pointers, is dropped (the next cfgpp_prepare
  // builds it), and the packed K‖V copies that read the key are re-packed in place
  const bool reload = weights_.has(key);
  if (reload) CFGPP_CHECK_CUDA(cudaDeviceSynchronize());  // a replay may still read the old tensor
  weights_.load(key, data, shape, ndim, dtype, stream);
  if (reload) {
    weights_.refresh({key}, stream);
    prepared_ = false;
    graph_valid_ = false;
    nsteps_ = 0;
  }
  ip_ready_ = false;
}

void Unet::ip_attach(int n_tokens, int embed_dim) {
  CFGPP_REQUIRE(!is_cn_, "an IP-Adapter attaches to a UNet handle, not a ControlNet");
  CFGPP_REQUIRE(finalized_, "call cfgpp_finalize_weights first");
  if (n_tokens != 0) {
    CFGPP_REQUIRE(n_tokens >= 1 && n_tokens <= 64, "an IP-Adapter has 1..64 image tokens");
    CFGPP_REQUIRE(embed_dim >= 8 && embed_dim % 8 == 0, "the image embedding width must be a positive multiple of 8");
  }
  ip_ntok_ = n_tokens;
  ip_embed_dim_ = n_tokens ? embed_dim : 0;
  ip_rs_ = cfgpp_ip_resampler_desc{};  // ip_attach_resampler sets it after this call
  // the plan changes shape: the next cfgpp_prepare builds it
  prepared_ = false;
  graph_valid_ = false;
  nsteps_ = 0;
  ip_ready_ = false;
}

void Unet::set_ip_image_embeds(const __half* embeds, cudaStream_t stream) {
  CFGPP_REQUIRE(ip_ntok_ > 0, "no IP-Adapter attached");
  CFGPP_REQUIRE(ip_rs_.num_queries == 0, "the attached IP-Adapter Plus takes the image encoder's hidden states "
                                         "(cfgpp_set_ip_image_hidden_states), not image embeds");
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(embeds != nullptr, "null image embeds");
  CFGPP_CHECK_CUDA(cudaMemcpyAsync(ip_embeds_, embeds, static_cast<size_t>(NB_) * ip_embed_dim_ * sizeof(__half),
                                   cudaMemcpyDeviceToDevice, stream));
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  run_plan(ip_plan_, stream);
  ip_ready_ = true;
}

void Unet::set_ip_scale(float scale, cudaStream_t stream) {
  CFGPP_REQUIRE(!is_cn_, "the IP-Adapter scale is set on the UNet handle");
  ip_scale_ = scale;
  // pageable source: staged before the call returns; the stream orders it after a replay still reading the word
  if (prepared_)
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(&args_->ip_scale, &ip_scale_, sizeof(float), cudaMemcpyHostToDevice, stream));
}

// ------------------------------------------------------------------------------------------------------------
// T2I-Adapter
// ------------------------------------------------------------------------------------------------------------
void Unet::t2i_attach(int n_features) {
  CFGPP_REQUIRE(!is_cn_, "T2I-Adapter features attach to a UNet handle, not a ControlNet");
  const int L = d_.num_levels;
  // the last down block has no downsampler, so the mid-block output always has its shape: an (L+1)-th feature lands
  // there
  CFGPP_REQUIRE(n_features == 0 || n_features == L || n_features == L + 1,
                "a T2I-Adapter for this UNet has num_levels (" + std::to_string(L) + ") or num_levels + 1 features, "
                "not " + std::to_string(n_features));
  t2i_n_ = n_features;
  // the plan changes shape: the next cfgpp_prepare builds it
  prepared_ = false;
  graph_valid_ = false;
  nsteps_ = 0;
  t2i_ready_ = false;
}

void Unet::set_t2i_features(const __half* const* features, cudaStream_t stream) {
  CFGPP_REQUIRE(t2i_n_ > 0, "no T2I-Adapter features attached (cfgpp_t2i_attach)");
  CFGPP_REQUIRE(prepared_, "call cfgpp_prepare first");
  CFGPP_REQUIRE(features != nullptr, "null feature table");
  for (int k = 0; k < t2i_n_; ++k) CFGPP_REQUIRE(features[k] != nullptr, "null T2I feature");
  for (int k = 0; k < t2i_n_; ++k)
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(t2i_feat_[k].p, features[k],
                                     static_cast<size_t>(B_) * t2i_hw_[k] * t2i_feat_[k].C * sizeof(__half),
                                     cudaMemcpyDeviceToDevice, stream));
  t2i_ready_ = true;
}

void Unet::set_t2i_active(int on, cudaStream_t stream) {
  CFGPP_REQUIRE(!is_cn_, "the T2I word is set on the UNet handle");
  t2i_on_ = on ? 1 : 0;
  for (StepEntry& e : entries_) e.t2i_on = t2i_on_;
  if (prepared_ && nsteps_ > 0) upload_entries(stream);
}

void Unet::set_t2i_steps(const int* on, int n, cudaStream_t stream) {
  CFGPP_REQUIRE(prepared_ && nsteps_ > 0, "call cfgpp_set_schedule first");
  CFGPP_REQUIRE(on != nullptr && n == nsteps_, "one T2I word per schedule entry");
  for (int i = 0; i < n; ++i) entries_[i].t2i_on = on[i] ? 1 : 0;
  upload_entries(stream);
}

void Unet::cond_embed(const void* image, int is_half, int B, int Hi, int Wi, __half* out, cudaStream_t stream) {
  CFGPP_REQUIRE(is_cn_ && finalized_, "the conditioning embedding runs on a finalized ControlNet handle");
  CFGPP_REQUIRE(image != nullptr && out != nullptr, "null argument");
  const int n = cn_desc_.num_embedding_levels;
  const int f = 1 << (n - 1);
  CFGPP_REQUIRE(B >= 1 && B <= 8 && Hi >= f && Wi >= f && Hi % f == 0 && Wi % f == 0,
                "control image: batch 1..8, height and width multiples of 8");
  // every intermediate is NHWC with its channels zero-padded to the convolution's 64-wide K blocks; two ping-pong
  // buffers sized for the largest, allocated for this call only (the embedding runs once per image, not per step)
  const EmbedConv& in = embed_convs_.at("conv_in");
  size_t need = static_cast<size_t>(B) * Hi * Wi * std::max(in.cin_p, in.cout_p);
  for (int i = 0; i + 1 < n; ++i) {
    const EmbedConv& s2 = embed_convs_.at("blocks." + std::to_string(2 * i + 1));
    need = std::max(need, static_cast<size_t>(B) * (Hi >> i) * (Wi >> i) * s2.cin_p);
    need = std::max(need, static_cast<size_t>(B) * (Hi >> (i + 1)) * (Wi >> (i + 1)) * s2.cout_p);
  }
  __half *a = nullptr, *b = nullptr;
  CFGPP_CHECK_CUDA(cudaMallocAsync(&a, need * sizeof(__half), stream));
  CFGPP_CHECK_CUDA(cudaMallocAsync(&b, need * sizeof(__half), stream));
  try {
    run_image_to_nhwc(image, is_half, a, B, cn_desc_.conditioning_channels, Hi, Wi, in.cin_p, stream);
    int h = Hi, w = Wi;
    auto conv = [&](const std::string& name, const __half* x, __half* y, int stride, bool silu) {
      const EmbedConv& c = embed_convs_.at(name);
      run_gemm_op(make_conv3x3_op(x, B, h, w, c.cin_p, c.w, c.cout_p, c.b, nullptr, 0, 1, y, 0, stride), stream);
      h /= stride;
      w /= stride;
      if (silu) run_silu(y, static_cast<size_t>(B) * h * w * c.cout_p, stream);
    };
    conv("conv_in", a, b, 1, true);
    for (int i = 0; i + 1 < n; ++i) {
      conv("blocks." + std::to_string(2 * i), b, a, 1, true);
      conv("blocks." + std::to_string(2 * i + 1), a, b, 2, true);
    }
    conv("conv_out", b, out, 1, false);
  } catch (...) {
    cudaFreeAsync(a, stream);
    cudaFreeAsync(b, stream);
    throw;
  }
  CFGPP_CHECK_CUDA(cudaFreeAsync(a, stream));
  CFGPP_CHECK_CUDA(cudaFreeAsync(b, stream));
}

}  // namespace cfgpp
