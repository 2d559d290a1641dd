// cfgpp_b200 — AutoencoderKL DECODER executor (SURVEY.md §8 f2): `vae.decode(zt / scaling_factor).sample` of the
// reference (latent_sdxl.py:155-164 with madebyollin/sdxl-vae-fp16-fix :44; latent_diffusion.py:123-129) on the
// UNet's kernels: implicit-GEMM conv3x3 and 1x1 / linear GEMMs on wgmma, GroupNorm(+SiLU), nearest-2x upsample,
// conv_in (4 -> C) — plus the three small kernels of vae_kernels.cu. Structure = diffusers 0.27.1 `Decoder`:
//   post_quant_conv 1x1 -> conv_in -> mid_block (resnet, single-head attention over all H*W tokens, resnet)
//   -> up_blocks (layers_per_block + 1 resnets each, nearest-2x + conv between levels) -> GroupNorm + SiLU -> conv_out.
// Activations are NHWC fp16 (tokens x channels), the image leaves as NCHW fp16 (the caller's `.float()` follows).
// The single-head attention has head dim = C (512): S = Q K^T and O = P V run as two GEMMs with a row-softmax pass
// in between (the score matrix is materialised: N x N fp16, 512 MB at 128 x 128 latents, one sample at a time).
#pragma once
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/cfgpp_b200.h"
#include "executor.cuh"
#include "gemm.cuh"
#include "ops.cuh"

namespace cfgpp {

// vae_kernels.cu
void run_vae_latent_prep(const void* z, int z_is_half, float scaling, const __half* w, const __half* bias, __half* out,
                         int B, int HW, cudaStream_t stream);
void run_vae_row_softmax(__half* s, int rows, int n, float scale_log2e, cudaStream_t stream);
void run_vae_conv_rgb(const __half* x, const __half* w, const __half* bias, __half* out, int B, int H, int W, int C,
                      cudaStream_t stream);
void run_vae_image_pad(const void* x, int x_is_half, __half* out, int B, int H, int W, cudaStream_t stream);
void run_vae_moments_sample(const __half* x, const __half* w, const __half* bias, const __half* wq, const __half* bq,
                            const __half* noise, float scaling, float* out, int B, int H, int W, int C,
                            cudaStream_t stream);

class VaeDecoder {
 public:
  VaeDecoder(const cfgpp_vae_desc& d, int device);
  void load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                   cudaStream_t stream);
  void finalize_weights(cudaStream_t stream);
  // z: (batch, 4, h, w) NCHW of z_dtype (the scaled latent zt); image: (batch, 3, 8h.., 8w..) NCHW fp16
  void decode(const void* z, int z_dtype, int batch, int h_lat, int w_lat, __half* image, cudaStream_t stream);
  // ENCODER half (`vae.encode(x).latent_dist.sample() * scaling_factor`, latent_sdxl.py:151-152, latent_diffusion.py:
  // 117-121; weights `encoder.*`, `quant_conv.*`): image (batch,3,H,W) NCHW of x_dtype -> scaled latent (batch,4,H/8,W/8)
  // fp32 (what the fp16 module returns under the reference's autocast). noise: the caller's `randn(mean.shape)` draw in fp16, or null for the posterior mean.
  void encode(const void* image, int x_dtype, int batch, int H, int W, const __half* noise, float* latent,
              cudaStream_t stream);
  bool has_encoder() const { return weights_.has("encoder.conv_in.weight"); }
  double encode_flops() const { return enc_.flops; }
  double flops() const { return dec_.flops; }
  size_t workspace_bytes() const { return dec_.arena.bytes(); }  // one decode of the prepared shape

 private:
  // one direction's launch plan for its prepared shape, with the workspace it runs in
  struct Plan {
    std::vector<std::function<void(cudaStream_t)>> steps;
    double flops = 0.0;
    DeviceArena arena;
    int batch = 0, h = 0, w = 0;  // batch 0: nothing prepared
  };
  void begin_plan(Plan& plan);
  __half* alloc_act(size_t numel) { return cur_->arena.alloc<__half>(numel); }
  void prepare(int batch, int h_lat, int w_lat);
  void prepare_encode(int batch, int H, int W);
  void add(std::function<void(cudaStream_t)> fn) { cur_->steps.push_back(std::move(fn)); }
  void add_gemm(const GemmOp& op) {
    cur_->flops += op.flops();
    cur_->steps.push_back([op](cudaStream_t st) { run_gemm_op(op, st); });
  }
  void alloc_scratch(size_t max_act, size_t ntok, int Ct);  // the builders' scratch set, into the current plan's arena
  // builders return the output activation pointer
  __half* build_resnet(const std::string& prefix, const __half* x, int Cin, int Cout, int H, int W);
  __half* build_attention(const std::string& prefix, const __half* x, int C, int H, int W);
  __half* next_out();

  cfgpp_vae_desc d_;
  int device_;
  bool finalized_ = false;
  WeightStore weights_;
  StreamKWorkspace sk_;
  Plan dec_, enc_;    // decode (latent shape), encode (image shape)
  Plan* cur_ = &dec_;  // the plan the builders append to
  int nb_ = 0;                     // batch the builders lay the current plan out for
  const void* x_in_ = nullptr;     // set per encode() call
  int x_is_half_ = 0;
  const __half* noise_in_ = nullptr;
  float* latent_out_ = nullptr;
  __half* conv_in_w4_ = nullptr;   // encoder.conv_in.weight (C,3,3,3) zero-padded to (C,4,3,3)
  const void* z_in_ = nullptr;   // set per decode() call (read by the first plan step through these members)
  int z_is_half_ = 0;
  __half* image_out_ = nullptr;
  // workspace
  __half* rot_[3] = {nullptr, nullptr, nullptr};  // rotating block outputs
  int rot_i_ = 0;
  __half *s_norm_ = nullptr, *s_h1_ = nullptr, *s_sc_ = nullptr, *s_up_ = nullptr, *zq_ = nullptr;
  __half *s_q_ = nullptr, *s_k_ = nullptr, *s_vt_ = nullptr, *s_scores_ = nullptr, *s_o_ = nullptr;
  float* gn_partial_ = nullptr;
};

}  // namespace cfgpp
