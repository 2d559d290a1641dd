// cfgpp_b200 — AutoencoderKL decoder executor (see vae.cuh). Host-side orchestration only.
#include "vae.cuh"

#include <algorithm>
#include <cmath>

namespace cfgpp {

void gemm_configure();

VaeDecoder::VaeDecoder(const cfgpp_vae_desc& d, int device) : d_(d), device_(device), sk_(device) {
  CFGPP_CHECK_CUDA(cudaSetDevice(device));
  CFGPP_REQUIRE(d.num_levels >= 2 && d.num_levels <= CFGPP_MAX_LEVELS, "num_levels must be 2..4");
  CFGPP_REQUIRE(d.latent_channels == 4 && d.out_channels == 3, "the decoder maps 4 latent channels to 3 image channels");
  CFGPP_REQUIRE(d.norm_num_groups == 32, "only GroupNorm(32) is implemented");
  for (int i = 0; i < d.num_levels; ++i)
    CFGPP_REQUIRE(d.block_out_channels[i] % 64 == 0, "decoder channel counts must be multiples of 64");
  CFGPP_REQUIRE(d.scaling_factor > 0.f, "scaling_factor must be positive");
  gemm_configure();
}

void VaeDecoder::load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                             cudaStream_t stream) {
  CFGPP_REQUIRE(!finalized_, "weights already finalized");
  weights_.load(key, data, shape, ndim, dtype, stream);
}

void VaeDecoder::finalize_weights(cudaStream_t stream) {
  CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));
  finalized_ = true;
  try {  // structural validation: a dry plan at the smallest latent touches (and packs) every weight
    prepare(1, 16, 16);
    if (has_encoder()) {
      const WeightStore::Weight& ci = weights_.raw("encoder.conv_in.weight");
      CFGPP_REQUIRE(ci.shape.size() == 4 && ci.shape[1] == 3 && ci.shape[2] == 3 && ci.shape[3] == 3 &&
                        ci.shape[0] == d_.block_out_channels[0],
                    "encoder.conv_in.weight must be (C0,3,3,3)");
      conv_in_w4_ = weights_.packed_heads_cols("encoder.conv_in.weight", 1, 27, 36);
      prepare_encode(1, 128, 128);
    }
  } catch (...) {
    finalized_ = false;
    throw;
  }
}

// drops `plan` (launches and workspace) and makes it the one the builders append to
void VaeDecoder::begin_plan(Plan& plan) {
  plan.steps.clear();
  plan.arena.clear();
  plan.flops = 0.0;
  plan.batch = 0;
  cur_ = &plan;
}

__half* VaeDecoder::next_out() {
  rot_i_ = (rot_i_ + 1) % 3;
  return rot_[rot_i_];
}

// ResnetBlock2D without time embedding (eps 1e-6): GN+SiLU -> conv3x3 -> GN+SiLU -> conv3x3 (+ x or 1x1 shortcut)
__half* VaeDecoder::build_resnet(const std::string& prefix, const __half* x, int Cin, int Cout, int H, int W) {
  const int HW = H * W, NB = nb_;
  const int M = NB * HW;
  const __half *g1 = weights_.plain(prefix + ".norm1.weight"), *b1 = weights_.plain(prefix + ".norm1.bias");
  const __half *g2 = weights_.plain(prefix + ".norm2.weight"), *b2 = weights_.plain(prefix + ".norm2.bias");
  __half *normp = s_norm_, *h1 = s_h1_;
  float* partial = gn_partial_;
  add([=](cudaStream_t st) { run_groupnorm(x, Cin, nullptr, 0, NB, HW, g1, b1, 1e-6f, true, partial, normp, st); });
  add_gemm(make_conv3x3_op(normp, NB, H, W, Cin, weights_.packed_conv3x3(prefix + ".conv1.weight"), Cout, weights_.plain(prefix + ".conv1.bias"),
                           nullptr, 0, 1, h1));
  add([=](cudaStream_t st) { run_groupnorm(h1, Cout, nullptr, 0, NB, HW, g2, b2, 1e-6f, true, partial, normp, st); });
  const __half* residual = x;
  if (Cin != Cout) {
    add_gemm(make_linear_op(x, Cin, nullptr, 0, 0, weights_.plain(prefix + ".conv_shortcut.weight"), M, Cout, Cin,
                            weights_.plain(prefix + ".conv_shortcut.bias"), nullptr, 0, 1, s_sc_, Cout, false));
    residual = s_sc_;
  }
  __half* out = next_out();
  add_gemm(make_conv3x3_op(normp, NB, H, W, Cout, weights_.packed_conv3x3(prefix + ".conv2.weight"), Cout, weights_.plain(prefix + ".conv2.bias"),
                           residual, Cout, 1, out));
  return out;
}

// UNetMidBlock2D attention (one head of width C over all H*W tokens, biased projections, residual connection)
__half* VaeDecoder::build_attention(const std::string& prefix, const __half* x, int C, int H, int W) {
  const int N = H * W, NB = nb_;
  CFGPP_REQUIRE(N % 64 == 0, "mid-block attention needs H*W to be a multiple of 64");
  const __half *g = weights_.plain(prefix + ".group_norm.weight"), *b = weights_.plain(prefix + ".group_norm.bias");
  __half *normp = s_norm_, *q = s_q_, *k = s_k_, *vt = s_vt_, *sc = s_scores_, *o = s_o_;
  float* partial = gn_partial_;
  add([=](cudaStream_t st) { run_groupnorm(x, C, nullptr, 0, NB, N, g, b, 1e-6f, false, partial, normp, st); });
  add_gemm(make_linear_op(normp, C, nullptr, 0, 0, weights_.plain(prefix + ".to_q.weight"), NB * N, C, C, weights_.plain(prefix + ".to_q.bias"),
                          nullptr, 0, 1, q, C, false));
  add_gemm(make_linear_op(normp, C, nullptr, 0, 0, weights_.plain(prefix + ".to_k.weight"), NB * N, C, C, weights_.plain(prefix + ".to_k.bias"),
                          nullptr, 0, 1, k, C, false));
  const float scale_log2e = (1.0f / sqrtf(static_cast<float>(C))) * 1.4426950408889634f;
  const __half *wv = weights_.plain(prefix + ".to_v.weight"), *bv = weights_.plain(prefix + ".to_v.bias");
  for (int s = 0; s < NB; ++s) {  // the N x N score matrix is materialised one sample at a time
    const __half* qs = q + static_cast<size_t>(s) * N * C;
    const __half* ks = k + static_cast<size_t>(s) * N * C;
    const __half* ns = normp + static_cast<size_t>(s) * N * C;
    __half* os = o + static_cast<size_t>(s) * N * C;
    // S = Q K^T                                   [N x N]
    add_gemm(make_linear_op(qs, C, nullptr, 0, 0, ks, N, N, C, nullptr, nullptr, 0, 1, sc, N, false));
    add([=](cudaStream_t st) { run_vae_row_softmax(sc, N, N, scale_log2e, st); });
    // V0^T = Wv X^T (no bias)                      [C x N]: the MN-major operand the P V GEMM needs as its "weight"
    add_gemm(make_linear_op(wv, C, nullptr, 0, 0, ns, C, N, C, nullptr, nullptr, 0, 1, vt, N, false));
    // O = P V0 + b_v (rows of P sum to 1, so the value bias commutes with the softmax average)   [N x C]
    add_gemm(make_linear_op(sc, N, nullptr, 0, 0, vt, N, C, N, bv, nullptr, 0, 1, os, C, false));
  }
  __half* out = next_out();
  add_gemm(make_linear_op(o, C, nullptr, 0, 0, weights_.plain(prefix + ".to_out.0.weight"), NB * N, C, C,
                          weights_.plain(prefix + ".to_out.0.bias"), x, C, 1, out, C, false));
  return out;
}

void VaeDecoder::alloc_scratch(size_t max_act, size_t ntok, int Ct) {
  const size_t NB = nb_;
  for (int i = 0; i < 3; ++i) rot_[i] = alloc_act(NB * max_act);
  rot_i_ = 0;
  s_norm_ = alloc_act(NB * max_act);
  s_h1_ = alloc_act(NB * max_act);
  s_sc_ = alloc_act(NB * max_act);
  s_q_ = alloc_act(NB * ntok * Ct);
  s_k_ = alloc_act(NB * ntok * Ct);
  s_o_ = alloc_act(NB * ntok * Ct);
  s_vt_ = alloc_act(ntok * Ct);
  s_scores_ = alloc_act(ntok * ntok);
  gn_partial_ = cur_->arena.alloc<float>(NB * 128 * 64);
}

void VaeDecoder::prepare(int batch, int h_lat, int w_lat) {
  CFGPP_REQUIRE(finalized_, "call cfgpp_vae_finalize_weights first");
  CFGPP_REQUIRE(batch >= 1 && batch <= 16, "decode batch must be 1..16");
  CFGPP_REQUIRE(h_lat >= 8 && w_lat >= 8 && (h_lat * w_lat) % 64 == 0, "latent H * W must be a multiple of 64");
  const int L = d_.num_levels;
  bool tiled = true;  // every level tiled-addressable, or a latent of at least 64 x 64 (im2col A tiles elsewhere)
  for (int i = 0, h = h_lat, w = w_lat; i < L; ++i, h *= 2, w *= 2) tiled = tiled && conv3x3_geometry_supported(h, w);
  CFGPP_REQUIRE(tiled || latent_allows_im2col(h_lat, w_lat),
                "latent " + std::to_string(h_lat) + "x" + std::to_string(w_lat) +
                    ": a latent whose decoder levels are not all tiled-addressable must be at least 64 x 64 (512 px images)");
  CFGPP_CHECK_CUDA(cudaSetDevice(device_));
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
  StreamKScope sk_scope(sk_.ws(), sk_.flags());  // the decoder's GEMM ops use its own stream-K workspace
  begin_plan(dec_);
  const int NB = batch;
  nb_ = NB;
  // sizes: the largest activation of the walk (elements per sample)
  size_t max_act = 0;
  {
    int h = h_lat, w = w_lat, c = d_.block_out_channels[L - 1];
    max_act = static_cast<size_t>(h) * w * c;
    for (int i = 0; i < L; ++i) {
      const int cout = d_.block_out_channels[L - 1 - i];
      max_act = std::max(max_act, static_cast<size_t>(h) * w * std::max(c, cout));
      c = cout;
      if (i != L - 1) {
        h *= 2;
        w *= 2;
        max_act = std::max(max_act, static_cast<size_t>(h) * w * c);  // upsampled tensor and its conv output
      }
    }
  }
  const int Ct = d_.block_out_channels[L - 1];
  const size_t ntok = static_cast<size_t>(h_lat) * w_lat;
  alloc_scratch(max_act, ntok, Ct);
  s_up_ = alloc_act(NB * max_act);
  zq_ = alloc_act(static_cast<size_t>(NB) * 4 * h_lat * w_lat);

  // ---- plan ----
  const float scaling = d_.scaling_factor;
  const __half *wpq = weights_.plain("post_quant_conv.weight"), *bpq = weights_.plain("post_quant_conv.bias");
  const __half *wci = weights_.plain("decoder.conv_in.weight"), *bci = weights_.plain("decoder.conv_in.bias");
  CFGPP_REQUIRE(weights_.raw("post_quant_conv.weight").numel() == 16, "post_quant_conv must be a 4 -> 4 1x1 convolution");
  __half* zq = zq_;
  __half* x0 = rot_[0];
  const int h0 = h_lat, w0 = w_lat;
  add([=](cudaStream_t st) {
    run_vae_latent_prep(z_in_, z_is_half_, scaling, wpq, bpq, zq, NB, h0 * w0, st);
    run_conv_in(zq, 1, nullptr, wci, bci, x0, NB, h0, w0, Ct, 1, st);
  });
  dec_.flops += 2.0 * NB * h0 * w0 * 36.0 * Ct;
  const __half* x = x0;
  x = build_resnet("decoder.mid_block.resnets.0", x, Ct, Ct, h0, w0);
  x = build_attention("decoder.mid_block.attentions.0", x, Ct, h0, w0);
  x = build_resnet("decoder.mid_block.resnets.1", x, Ct, Ct, h0, w0);
  int H = h0, W = w0, C = Ct;
  for (int i = 0; i < L; ++i) {
    const int Cout = d_.block_out_channels[L - 1 - i];
    const std::string blk = "decoder.up_blocks." + std::to_string(i);
    for (int j = 0; j < d_.layers_per_block + 1; ++j) {
      x = build_resnet(blk + ".resnets." + std::to_string(j), x, C, Cout, H, W);
      C = Cout;
    }
    if (i != L - 1) {
      const __half* xin = x;
      __half* up = s_up_;
      const int Hc = H, Wc = W, Cc = C;
      add([=](cudaStream_t st) { run_upsample2x(xin, up, NB, Hc, Wc, Cc, st); });
      H *= 2;
      W *= 2;
      __half* out = next_out();
      add_gemm(make_conv3x3_op(up, NB, H, W, C, weights_.packed_conv3x3(blk + ".upsamplers.0.conv.weight"), C,
                               weights_.plain(blk + ".upsamplers.0.conv.bias"), nullptr, 0, 1, out));
      x = out;
    }
  }
  {
    const __half *g = weights_.plain("decoder.conv_norm_out.weight"), *b = weights_.plain("decoder.conv_norm_out.bias");
    const __half* wco = weights_.packed_conv3x3("decoder.conv_out.weight");
    const __half* bco = weights_.plain("decoder.conv_out.bias");
    CFGPP_REQUIRE(weights_.raw("decoder.conv_out.weight").shape[0] == 3, "conv_out must produce 3 channels");
    __half* normp = s_norm_;
    float* partial = gn_partial_;
    const __half* xin = x;
    const int Hc = H, Wc = W, Cc = C;
    add([=](cudaStream_t st) {
      run_groupnorm(xin, Cc, nullptr, 0, NB, Hc * Wc, g, b, 1e-6f, true, partial, normp, st);
      run_vae_conv_rgb(normp, wco, bco, image_out_, NB, Hc, Wc, Cc, st);
    });
    dec_.flops += 2.0 * NB * Hc * Wc * 27.0 * Cc;
  }
  dec_.batch = NB; dec_.h = h_lat; dec_.w = w_lat;
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
}

void VaeDecoder::decode(const void* z, int z_dtype, int batch, int h_lat, int w_lat, __half* image,
                        cudaStream_t stream) {
  CFGPP_REQUIRE(z_dtype == CFGPP_F16 || z_dtype == CFGPP_F32, "latent dtype must be fp16 or fp32");
  if (batch != dec_.batch || h_lat != dec_.h || w_lat != dec_.w) prepare(batch, h_lat, w_lat);
  z_in_ = z;
  z_is_half_ = (z_dtype == CFGPP_F16) ? 1 : 0;
  image_out_ = image;
  for (auto& fn : dec_.steps) fn(stream);
}

// ---- encoder ----------------------------------------------------------------------------------------------------
// diffusers 0.27.1 `Encoder` + quant_conv + DiagonalGaussianDistribution.sample: conv_in (3 -> C0) -> down_blocks
// (layers_per_block resnets each; Downsample2D = zero row / column after the image + stride-2 conv, as an implicit GEMM
// through a stride-2 tensor map that starts at the pixel itself) -> mid_block -> GroupNorm + SiLU -> conv_out (8
// moments) -> quant_conv 1x1 -> mean + std * noise, times scaling_factor.
void VaeDecoder::prepare_encode(int batch, int H, int W) {
  CFGPP_REQUIRE(finalized_, "call cfgpp_vae_finalize_weights first");
  CFGPP_REQUIRE(has_encoder() && conv_in_w4_ != nullptr, "this handle holds no encoder weights (encoder.*, quant_conv.*)");
  CFGPP_REQUIRE(batch >= 1 && batch <= 16, "encode batch must be 1..16");
  const int L = d_.num_levels;
  const int f = 1 << (L - 1);
  CFGPP_REQUIRE(H >= 8 * f && W >= 8 * f && H % f == 0 && W % f == 0, "image size must be a multiple of the VAE factor");
  CFGPP_REQUIRE(((H / f) * (W / f)) % 64 == 0, "latent H * W must be a multiple of 64");
  bool tiled = true;  // every level tiled-addressable, or a latent of at least 64 x 64 (im2col A tiles elsewhere)
  for (int i = 0, h = H, w = W; i < L; ++i, h /= 2, w /= 2) {
    CFGPP_REQUIRE(w % 4 == 0, "encoder level width " + std::to_string(w) + " must be a multiple of 4");
    tiled = tiled && conv3x3_geometry_supported(h, w);
  }
  CFGPP_REQUIRE(tiled || latent_allows_im2col(H / f, W / f),
                "image " + std::to_string(H) + "x" + std::to_string(W) +
                    ": an image whose encoder levels are not all tiled-addressable must be at least 512 x 512 px");
  CFGPP_CHECK_CUDA(cudaSetDevice(device_));
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
  StreamKScope sk_scope(sk_.ws(), sk_.flags());
  begin_plan(enc_);
  const int NB = batch;
  nb_ = NB;
  size_t max_act = 0;
  {
    int h = H, w = W, c = d_.block_out_channels[0];
    max_act = static_cast<size_t>(h) * w * c;
    for (int i = 0; i < L; ++i) {
      c = std::max(c, d_.block_out_channels[i]);
      max_act = std::max(max_act, static_cast<size_t>(h) * w * c);
      if (i != L - 1) { h /= 2; w /= 2; }
    }
  }
  const int Ct = d_.block_out_channels[L - 1];
  const int hl = H / f, wl = W / f;
  alloc_scratch(max_act, static_cast<size_t>(hl) * wl, Ct);
  __half* img4 = alloc_act(static_cast<size_t>(NB) * 4 * H * W);

  const int C0 = d_.block_out_channels[0];
  const __half* wci = conv_in_w4_;
  const __half* bci = weights_.plain("encoder.conv_in.bias");
  __half* x0 = rot_[0];
  add([=](cudaStream_t st) {
    run_vae_image_pad(x_in_, x_is_half_, img4, NB, H, W, st);
    run_conv_in(img4, 1, nullptr, wci, bci, x0, NB, H, W, C0, 1, st);
  });
  enc_.flops += 2.0 * NB * H * W * 27.0 * C0;
  const __half* x = x0;
  int h = H, w = W, C = C0;
  for (int i = 0; i < L; ++i) {
    const int Cout = d_.block_out_channels[i];
    const std::string blk = "encoder.down_blocks." + std::to_string(i);
    for (int j = 0; j < d_.layers_per_block; ++j) {
      x = build_resnet(blk + ".resnets." + std::to_string(j), x, C, Cout, h, w);
      C = Cout;
    }
    if (i != L - 1) {
      __half* out = next_out();
      add_gemm(make_conv3x3_op(x, NB, h, w, C, weights_.packed_conv3x3(blk + ".downsamplers.0.conv.weight"), C,
                               weights_.plain(blk + ".downsamplers.0.conv.bias"), nullptr, 0, 1, out, 0, /*stride=*/2, /*pad=*/0));
      x = out;
      h /= 2;
      w /= 2;
    }
  }
  x = build_resnet("encoder.mid_block.resnets.0", x, C, C, h, w);
  x = build_attention("encoder.mid_block.attentions.0", x, C, h, w);
  x = build_resnet("encoder.mid_block.resnets.1", x, C, C, h, w);
  {
    const __half *g = weights_.plain("encoder.conv_norm_out.weight"), *b = weights_.plain("encoder.conv_norm_out.bias");
    const WeightStore::Weight& wo = weights_.raw("encoder.conv_out.weight");
    CFGPP_REQUIRE(wo.shape.size() == 4 && wo.shape[0] == 8 && wo.shape[1] == C, "encoder.conv_out must produce 8 moments");
    CFGPP_REQUIRE(weights_.raw("quant_conv.weight").numel() == 64 && weights_.raw("quant_conv.bias").numel() == 8,
                  "quant_conv must be an 8 -> 8 1x1 convolution");
    const __half* wco = weights_.packed_conv3x3("encoder.conv_out.weight");
    const __half *bco = weights_.plain("encoder.conv_out.bias"), *wq = weights_.plain("quant_conv.weight"), *bq = weights_.plain("quant_conv.bias");
    __half* normp = s_norm_;
    float* partial = gn_partial_;
    const __half* xin = x;
    const int hc = h, wc = w, Cc = C;
    const float scaling = d_.scaling_factor;
    add([=](cudaStream_t st) {
      run_groupnorm(xin, Cc, nullptr, 0, NB, hc * wc, g, b, 1e-6f, true, partial, normp, st);
      run_vae_moments_sample(normp, wco, bco, wq, bq, noise_in_, scaling, latent_out_, NB, hc, wc, Cc, st);
    });
    enc_.flops += 2.0 * NB * hc * wc * 72.0 * Cc;
  }
  enc_.batch = NB; enc_.h = H; enc_.w = W;
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
}

void VaeDecoder::encode(const void* image, int x_dtype, int batch, int H, int W, const __half* noise, float* latent,
                        cudaStream_t stream) {
  CFGPP_REQUIRE(x_dtype == CFGPP_F16 || x_dtype == CFGPP_F32, "image dtype must be fp16 or fp32");
  CFGPP_REQUIRE(image != nullptr && latent != nullptr, "null image / latent pointer");
  if (batch != enc_.batch || H != enc_.h || W != enc_.w) prepare_encode(batch, H, W);
  x_in_ = image;
  x_is_half_ = (x_dtype == CFGPP_F16) ? 1 : 0;
  noise_in_ = noise;
  latent_out_ = latent;
  for (auto& fn : enc_.steps) fn(stream);
}

}  // namespace cfgpp
