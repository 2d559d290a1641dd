// cfgpp_b200 — CLIP text tower executor (SURVEY.md §8 f3): the prompt conditioning of the reference —
// `pipe.text_encoder(ids)[0]` (SD v1.5, latent_diffusion.py:93-115) and `text_enc(ids, output_hidden_states=True)` ->
// `hidden_states[-2]` / `[0]` for the two SDXL encoders (latent_sdxl.py:77-93) — i.e. transformers `CLIPTextModel` /
// `CLIPTextModelWithProjection`: token + position embedding, N pre-LN layers (causal self-attention with 64-wide
// heads, MLP with quick_gelu or gelu), final LayerNorm, pooled <|endoftext|> row (+ bias-free text_projection).
// Activations are [batch * tokens][hidden] fp16; the q/k/v projections run as ONE GEMM on a concatenated weight; every
// projection / MLP GEMM is the wgmma kernel of gemm.cu (residual adds in its epilogue), attention / activation /
// embedding are the kernels of text_kernels.cu, LayerNorm is norm.cu's.
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

// text_kernels.cu
void run_clip_embed(const int* ids, const __half* tok, const __half* pos, __half* out, int M, int T, int D, int vocab,
                    cudaStream_t stream);
void run_clip_attention(const __half* qkv, __half* out, int B, int T, int heads, int D, cudaStream_t stream);
void run_clip_activation(__half* x, size_t n, int mode, cudaStream_t stream);
void run_clip_gather_rows(const __half* x, const int* index, __half* out, int B, int T, int D, cudaStream_t stream);

// CLIP vision front end (text_kernels.cu): image [B,3,S,S] NCHW (fp16 or fp32) -> patch rows [B*(S/P)^2][Kp] fp16,
// row-major (channel, ky, kx) as conv2d's weight, columns 3*P*P..Kp-1 zero; and the embedding assembly
// x[b,0] = fp16(cls + pos[0]), x[b,1+p] = fp16(pe[b*np + p] + pos[1+p]).
void run_clip_patchify(const void* image, int is_half, __half* out, int B, int S, int P, int Kp, cudaStream_t stream);
void run_clip_vision_embed(const __half* pe, const __half* cls, const __half* pos, __half* out, int B, int np, int D,
                           cudaStream_t stream);

using ClipStep = std::function<void(cudaStream_t)>;
// The pre-LN encoder layer loop both CLIP towers share: per layer LN1 -> q|k|v GEMM -> attention -> out_proj (+ the
// residual, epilogue) -> LN2 -> fc1 -> activation -> fc2 (+ the residual). The towers differ only in the attention
// step (`attention`: qkv [M][3 * heads * hdp] -> att [M][heads * hdp]) and in the padded head width hdp the q|k|v and
// out_proj operands are packed with (the text tower's 64 is the plain concatenation and weight).
struct ClipLayerArgs {
  WeightStore* weights;
  std::string prefix;  // "<tower>.encoder.layers."
  int layers, D, I, M, act_mode;
  float eps;
  int heads, hdp;
  std::function<void(const __half* qkv, __half* att, cudaStream_t)> attention;
  double attention_flops;  // per layer
  __half *x0, *x1, *ln, *qkv, *att, *mlp;
};
std::vector<std::vector<ClipStep>> build_clip_layers(const ClipLayerArgs& a, double* flops);

class ClipTextEncoder {
 public:
  ClipTextEncoder(const cfgpp_clip_desc& d, int device);
  void load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                   cudaStream_t stream);
  void finalize_weights(cudaStream_t stream);
  // ids [batch][tokens] int32 (device), pooled_index [batch] int32 (device; may be null when pooled_out is null).
  // hidden_out = hidden_states[num_layers - skip] (no final LayerNorm), last_out = final_layer_norm(hidden_states[-1]),
  // pooled_out = last_out[b, pooled_index[b]] (x text_projection^T when projection_dim > 0). Null outputs are skipped.
  void encode(const int* ids, const int* pooled_index, int batch, int tokens, int skip, __half* hidden_out,
              __half* last_out, __half* pooled_out, cudaStream_t stream);
  double flops() const { return flops_; }
  size_t workspace_bytes() const { return act_.bytes(); }

 private:
  void prepare(int batch, int tokens);

  cfgpp_clip_desc d_;
  int device_;
  bool finalized_ = false;
  WeightStore weights_;
  DeviceArena act_;  // workspace of the prepared plan
  StreamKWorkspace sk_;
  double flops_ = 0.0;
  int B_ = 0, T_ = 0;
  std::vector<std::vector<ClipStep>> layer_plan_;  // one group of launches per encoder layer
  const int* ids_in_ = nullptr;                 // set per encode() call
  __half *x0_ = nullptr, *x1_ = nullptr, *ln_ = nullptr, *qkv_ = nullptr, *att_ = nullptr, *mlp_ = nullptr;
  __half *last_ = nullptr, *pool_ = nullptr;
};

// transformers CLIPVisionModelWithProjection: patch embedding (a bias-free PxP stride-P conv, as an unfold and a
// GEMM), class token and position embedding, pre_layrnorm, the shared layer loop with non-causal attention on the flash
// kernel (heads zero-padded to a multiple of 64 columns), post_layernorm of the CLS row, visual_projection.
class ClipVisionEncoder {
 public:
  ClipVisionEncoder(const cfgpp_clip_vision_desc& d, int device);
  void load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                   cudaStream_t stream);
  void finalize_weights(cudaStream_t stream);
  // image [batch][3][S][S] (fp16 or fp32, normalised pixel values) -> image_embeds [batch][projection_dim] fp16
  void encode(const void* image, int is_half, int batch, __half* embeds_out, cudaStream_t stream);
  // the same image -> hidden_states[num_layers - skip] [batch][T][hidden_size] fp16 (no post_layernorm; skip = 1 is
  // the penultimate layer IP-Adapter Plus reads); only the layers up to that one run
  void encode_hidden(const void* image, int is_half, int batch, int skip, __half* hidden_out, cudaStream_t stream);
  double flops() const { return flops_; }
  size_t workspace_bytes() const { return act_.bytes(); }

 private:
  void prepare(int batch);
  void embed(const void* image, int is_half, int batch, cudaStream_t stream);  // image -> hidden_states[0] in x0_

  cfgpp_clip_vision_desc d_;
  int device_;
  bool finalized_ = false;
  int T_ = 0, np_ = 0, Kp_ = 0, hdp_ = 0, Cp_ = 0;
  WeightStore weights_;
  DeviceArena act_;
  StreamKWorkspace sk_;
  __half* patch_w_ = nullptr;  // [D][Kp]
  double flops_ = 0.0;
  int B_ = 0;
  std::vector<std::vector<ClipStep>> layer_plan_;
  __half *patches_ = nullptr, *pe_ = nullptr, *emb_ = nullptr, *x0_ = nullptr, *x1_ = nullptr, *ln_ = nullptr,
         *qkv_ = nullptr, *att_ = nullptr, *mlp_ = nullptr, *cls_ = nullptr, *cls_ln_ = nullptr;
};

}  // namespace cfgpp
