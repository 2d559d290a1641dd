// cfgpp_b200 — UNet2DConditionModel executor: weights in a WeightStore, static launch plan over the hand-written
// kernels, CUDA-graph replay of one fused sampler step. Structure follows SURVEY.md Appendix A (diffusers 0.27.1).
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/cfgpp_b200.h"
#include "attention.cuh"
#include "executor.cuh"
#include "gemm.cuh"
#include "ops.cuh"

namespace cfgpp {

struct PlanStep {
  std::string name;
  double flops = 0.0;  // algorithmic FLOPs of this launch group (0 for non-contraction kernels)
  int launches = 1;
  int kind = 3;  // 0 linear GEMM, 1 conv3x3 (implicit GEMM), 2 attention, 3 other (norm / elementwise)
  std::function<void(cudaStream_t)> fn;
};

class Unet {
 public:
  // cn != null makes a ControlNet handle (diffusers ControlNetModel): the down / mid half of this class's plan on its
  // own weights, plus the conditioning embedding and the zero convs, run through the UNet handle it is attached to
  Unet(const cfgpp_model_desc& d, int device, const cfgpp_controlnet_desc* cn = nullptr);
  ~Unet();

  void load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                   cudaStream_t stream);
  void finalize_weights(cudaStream_t stream);
  // LoRA adapters (WeightStore::lora_*): factors are added per diffusers weight key after finalize; set_scales merges
  // every target from its pristine backup into the raw weight and re-runs the packers that read it, on `stream`. No
  // plan or graph pointer changes. The bound prompt goes stale (its K/V and add-embedding came from the old weights).
  void lora_add(int adapter, const std::string& key, const void* down, const void* up, int rank, float alpha, int dtype,
                cudaStream_t stream);
  void lora_set_scales(const float* scales_host, int n, cudaStream_t stream);
  void lora_clear(cudaStream_t stream);
  void lora_stats(int* n_adapters, int* n_targets, size_t* backup_bytes, size_t* bytes_moved) const;
  void prepare(int batch, int h_lat, int w_lat);
  // the prepared plan's workspace, the attached ControlNet's included
  size_t workspace_bytes() const { return act_.bytes() + (cn_ ? cn_->act_.bytes() : 0); }
  bool is_controlnet() const { return is_cn_; }
  double forward_flops() const { return forward_flops_; }
  int launches_per_step() const { return launches_per_step_; }
  double prompt_flops() const { return prompt_flops_; }
  int prompt_launches() const { return prompt_launches_; }
  int graph_captures() const { return graph_captures_; }  // step graphs captured over the handle's life

  void set_prompt(const __half* ctx, int n_ctx, const __half* pooled, const float* time_ids, int add_rows,
                  cudaStream_t stream);
  void unet_forward(const void* z, int z_dtype, float t, float in_scale, __half* eps_uc, __half* eps_c,
                    cudaStream_t stream);
  void set_schedule(int method, int state_dtype, const cfgpp_step_state* steps, int nsteps, cudaStream_t stream);
  void set_state(const void* z, int z_dtype, cudaStream_t stream);
  // ancestral samplers: fp16 noise table [slots][B,4,H,W] (device), copied into a handle-owned buffer
  void set_noise(const __half* noise, int slots, cudaStream_t stream);
  // per-image guidance: lambda_host [batch] (host), or n = 0 to return to the schedule's scalar; prepare() clears it
  void set_guidance(const float* lambda_host, int n, cudaStream_t stream);
  // v-prediction: (a, b) per entry of the current schedule (host [nsteps][2]); see cfgpp_set_v_coefs
  void set_v_coefs(const float* ab_host, int nsteps, cudaStream_t stream);
  void run_steps(int first_step, int nsteps, cudaStream_t stream);
  void get_state(int which, void* out, cudaStream_t stream);
  // ---- ControlNet (see cfgpp_attach_controlnet) ----
  void attach_controlnet(Unet* cn);  // UNet handles; null detaches
  void set_control_image(const void* image, int dtype, cudaStream_t stream);
  void set_control_scale(float scale, cudaStream_t stream);
  void set_control_scales(const float* scales_host, int n, cudaStream_t stream);
  // ControlNet handles: the conditioning embedding of image [B,3,Hi,Wi] -> out [B,Hi/8,Wi/8,C0] NHWC fp16
  void cond_embed(const void* image, int is_half, int B, int Hi, int Wi, __half* out, cudaStream_t stream);
  void apply_step(int step, const __half* eps_uc, const __half* eps_c, cudaStream_t stream);
  // ---- IP-Adapter (see cfgpp_ip_adapter_attach) ----
  void ip_load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                      cudaStream_t stream);
  void ip_attach(int n_tokens, int embed_dim);  // n_tokens = 0 detaches
  void set_ip_image_embeds(const __half* embeds, cudaStream_t stream);
  // IP-Adapter Plus (ip_resampler.cu): the Resampler image projection over hidden states [2*batch][seq_len][E]
  void ip_attach_resampler(const cfgpp_ip_resampler_desc& r);
  void set_ip_image_hidden_states(const __half* hidden, cudaStream_t stream);
  // Test and measurement aid: the image projection alone (the `image_proj.*` entries of the plan, on the image rows
  // already set), and a copy of its tokens [2*batch * n_tokens][D] into tokens_out (may be null)
  void run_image_proj(__half* tokens_out, cudaStream_t stream);
  void set_ip_scale(float scale, cudaStream_t stream);
  // ---- T2I-Adapter (see cfgpp_t2i_attach) ----
  void t2i_attach(int n_features);  // 0 detaches
  void set_t2i_features(const __half* const* features, cudaStream_t stream);
  void set_t2i_active(int on, cudaStream_t stream);
  void set_t2i_steps(const int* on_host, int n, cudaStream_t stream);
  // Eager un-fused forward with a CUDA-event pair around every plan entry (profiling aid for bench.py).
  struct ProfEntry {
    std::string name;
    int kind;
    double flops;
    float ms;
  };
  std::vector<ProfEntry> profile_forward(const void* z, int z_dtype, float t, float in_scale, cudaStream_t stream);

 private:
  // ---- weights ----
  size_t lora_bytes_moved_ = 0;  // of the last lora_set_scales / lora_clear
  bool prompt_stale_ = false;    // weights changed under the bound prompt: set_prompt must run again
  void require_fresh_prompt() const;

  // ---- workspace ----
  __half* alloc_act(size_t numel) { return act_.alloc<__half>(numel); }
  struct Scratch {
    size_t need = 0;
    __half* p = nullptr;
  };
  // ---- plan building ----
  struct Act {
    __half* p;
    int C;
  };
  Act build_resnet(const std::string& prefix, Act x1, const Act* x2, int Cout, int H, int W, int temb_off);
  Act build_transformer(const std::string& prefix, Act x, int H, int W, int layers, int heads);
  Act build_downsample(const std::string& prefix, Act x, int H, int W);
  Act build_upsample(const std::string& prefix, Act x, int H, int W);
  void add_gemm(const std::string& name, const GemmOp& op, double algorithmic_flops = -1.0);
  void add_attn(const std::string& name, const AttnOp& op);
  void add_step(const std::string& name, std::function<void(cudaStream_t)> fn, int launches = 1);
  void run_plan(const std::vector<PlanStep>& plan, cudaStream_t stream);
  void run_body(cudaStream_t stream);
  // the structure walk of prepare() (both passes) for this handle alone; `shared_args` (ControlNet handles built for
  // a UNet): the UNet's step record, whose timestep and input scale the ControlNet reads
  void build(int batch, int h_lat, int w_lat, StepArgs* shared_args);
  void build_control_plan();  // UNet handles with a ControlNet: the zero convs into the skip tensors and mid output
  void account();             // FLOP / launch totals of the built plan (+ the attached ControlNet's)
  std::vector<std::string> zero_conv_keys() const;  // ControlNet handles: one per entry of res_
  // prologue(s) and conv_in(s) of one forward on input z
  void run_inputs(const void* z, int z_is_half, cudaStream_t stream);
  void require_control_ready() const;
  void require_ip_ready() const;
  void require_t2i_ready() const;
  // UNet handles with T2I features attached: the gated add of the next feature onto h (H x W), in body_plan_
  void add_t2i_feature(Act h, int H, int W);
  void build_ip_resampler();  // ip_plan_ of an attached Resampler (ip_resampler.cu)
  void require_resampler_weights(const cfgpp_ip_resampler_desc& r) const;
  void upload_entries(cudaStream_t stream);  // entries_ -> step_table_
  // the un-fused forward's current entry: timestep and input scale, no step, the scalar conditioning scale
  void stage_entry(float t, float in_scale, cudaStream_t stream);
  void ensure_graph(cudaStream_t stream);

  cfgpp_model_desc d_;
  int device_;
  bool finalized_ = false, prepared_ = false;
  WeightStore weights_;
  DeviceArena act_;  // workspace of the prepared plan
  StreamKWorkspace sk_;

  // packed weights: resolved lazily during plan building (finalize just validates + packs what is shape-independent)
  __half* temb_w_all_ = nullptr;  // [sumCout][time_embed_dim]
  __half* temb_b_all_ = nullptr;
  int temb_total_ = 0;
  std::vector<std::pair<std::string, int>> temb_order_;  // resnet prefix -> offset
  int time_embed_dim_ = 0;

  // plan
  int B_ = 0, NB_ = 0, H_ = 0, W_ = 0;
  bool sizing_ = false;  // prepare()'s first pass: records scratch sizes, allocates and pushes nothing
  std::vector<PlanStep>* cur_plan_ = nullptr;
  std::vector<PlanStep> prologue_plan_;  // timestep embedding -> temb for all resnets
  std::vector<PlanStep> body_plan_;      // conv_in output .. mid block
  std::vector<PlanStep> control_plan_;   // the attached ControlNet's zero convs, added into res_ in place
  std::vector<PlanStep> up_plan_;        // up blocks
  std::vector<PlanStep> tail_plan_;      // conv_norm_out + SiLU
  std::vector<PlanStep> prompt_plan_;    // cross-attention K/V projections + add-embedding
  double forward_flops_ = 0.0, prompt_flops_ = 0.0;
  int launches_per_step_ = 0, prompt_launches_ = 0;

  // scratch (sized as the max over all uses while building, allocated afterwards; closures hold Scratch*)
  std::map<std::string, std::unique_ptr<Scratch>> scratch_;
  Scratch* scratch(const std::string& name, size_t numel_half);

  // conditioning / per-step device state
  __half* ctx_copy_ = nullptr;
  int n_ctx_ = 77;
  __half* add_in_ = nullptr;    // [NB][proj_in_dim]
  __half* add_h1_ = nullptr;
  __half* aug_emb_ = nullptr;   // [NB][time_embed_dim]
  __half* pooled_copy_ = nullptr;
  float* time_ids_copy_ = nullptr;  // [NB][n_time_ids_]
  bool has_aug_ = false;
  int n_time_ids_ = 0;  // (projection_class_embeddings_input_dim - pooled_dim) / addition_time_embed_dim
  __half *t_sin_ = nullptr, *t_h1_ = nullptr, *emb_ = nullptr, *semb_ = nullptr, *temb_all_ = nullptr;
  float* gn_partial_ = nullptr;
  StepArgs* args_ = nullptr;          // device; a ControlNet handle's is its UNet's
  StepEntry* step_table_ = nullptr;   // device [1024]
  int* step_counter_ = nullptr;       // device
  int nsteps_ = 0, method_ = 0, state_dtype_ = CFGPP_F32;
  std::vector<StepEntry> entries_;    // host mirror of the current schedule's nsteps_ entries
  bool v_pred_ = false;               // d_.prediction_type == 1
  bool v_ready_ = false;              // set_v_coefs matched the current schedule
  void* z_state_ = nullptr;   // (B,4,H,W) fp32-sized buffer (holds fp16 or fp32)
  void* aux_state_ = nullptr;
  void* z0t_state_ = nullptr;
  __half* noise_buf_ = nullptr;          // owned, survives prepare(); re-allocated when a larger table arrives
  size_t noise_cap_ = 0;                 // elements
  float* lambda_buf_ = nullptr;          // [B] per-image guidance, workspace of the prepared plan
  __half *fwd_eps_uc_ = nullptr, *fwd_eps_c_ = nullptr;
  Act final_norm_{nullptr, 0};
  __half* conv_in_out_ = nullptr;
  __half *conv_in_w_ = nullptr, *conv_in_b_ = nullptr, *conv_out_w_ = nullptr, *conv_out_b_ = nullptr;

  // ControlNet
  bool is_cn_ = false;
  cfgpp_controlnet_desc cn_desc_{};
  Unet* cn_ = nullptr;     // UNet handles: the attached ControlNet
  Unet* owner_ = nullptr;  // ControlNet handles: the UNet it is attached to
  std::vector<Act> res_;   // the down path's skip tensors, then the mid-block output (recorded by build)
  std::vector<int> res_hw_;
  __half* cond_ = nullptr;  // ControlNet handles: the conditioning embedding [B,H,W,C0] of the prepared shape
  struct EmbedConv {
    __half *w, *b;  // [Cout_p][9][Cin_p], [Cout_p], zero-padded
    int cout_p, cin_p;
  };
  std::map<std::string, EmbedConv> embed_convs_;
  float cn_scale_ = 1.0f;
  bool cn_image_ready_ = false;

  // IP-Adapter: the image tokens image_proj(embeds) [NB * ip_ntok_][D] and, per attn2, their K‖V, projected by
  // ip_plan_ once per set_ip_image_embeds; every attn2 of the body runs the decoupled cross-attention kernel
  int ip_ntok_ = 0, ip_embed_dim_ = 0;  // ip_ntok_ = 0: no adapter attached
  float ip_scale_ = 1.0f;
  bool ip_ready_ = false;               // image embeds projected for the current plan and weights
  __half *ip_embeds_ = nullptr, *ip_proj_ = nullptr, *ip_tokens_ = nullptr;
  std::vector<PlanStep> ip_plan_;
  // IP-Adapter Plus: the Resampler's geometry (num_queries = 0: the plain projection, or none) and its input
  cfgpp_ip_resampler_desc ip_rs_{};
  __half* ip_hidden_ = nullptr;  // [NB * seq_len][E]

  // T2I-Adapter: t2i_n_ features (0: none), each a [B, HW, C] buffer of the prepared plan that one gated add per step
  // adds into its placement (the body walk of build records them in order)
  int t2i_n_ = 0;
  int t2i_on_ = 1;           // the word of the un-fused forward and of a new schedule's entries
  bool t2i_ready_ = false;   // features copied for the current plan
  std::vector<Act> t2i_feat_;
  std::vector<int> t2i_hw_;

  cudaGraph_t graph_ = nullptr;
  cudaGraphExec_t graph_exec_ = nullptr;
  bool graph_valid_ = false;
  int graph_captures_ = 0;
  cudaStream_t capture_stream_ = nullptr;
};

}  // namespace cfgpp
