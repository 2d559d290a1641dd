/* cfgpp_b200 — C ABI of the Blackwell-native CFG++ sampling hot path (libcfgpp_b200.so).
 *
 * The reference (CFGpp-diffusion/CFGpp) has no FFI: its extension point is the Python solver registry
 * (latent_diffusion.py:13-26, latent_sdxl.py:15-28) and, inside a solver, the seam
 *     predict_noise(zt, t, uc, c[, added_cond_kwargs]) -> (eps_uc, eps_c)          latent_diffusion.py:131-158
 *                                                                                 latent_sdxl.py:167-185
 * which calls diffusers' UNet2DConditionModel.forward, followed by the hand-written CFG++ update of each solver
 * (latent_diffusion.py:660-666, 904-908; latent_sdxl.py:738-744, 902-919). This library replaces exactly that:
 * the batched (uncond+cond) UNet forward plus the guidance mix and scheduler update, as hand-written sm_90a CUDA.
 * The Python mirror of the solver API (cfgpp_b200/latent_diffusion.py, latent_sdxl.py) binds these symbols with
 * ctypes; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions: every function returns 0 on success or a negative status; cfgpp_last_error() returns the message of
 * the calling thread's last failure. No C++ exception crosses the boundary. All pointers named *_dev are CUDA
 * device pointers owned by the caller; the library owns only the opaque handle, its packed-weight arena and its
 * activation workspace. All work is enqueued asynchronously on the given cudaStream_t (passed as void*), with no
 * internal host synchronisation on the hot path. A handle is not thread-safe; use one per (process, GPU).
 * Layouts at the boundary are the reference's: latents NCHW contiguous (fp32 or fp16), context (rows,77,D) fp16.
 */
#ifndef CFGPP_B200_H_
#define CFGPP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CFGPP_MAX_LEVELS 4

/* UNet2DConditionModel structure (diffusers config fields; SURVEY.md Appendix A.1). */
typedef struct cfgpp_model_desc {
  int in_channels;                         /* 4 */
  int out_channels;                        /* 4 */
  int num_levels;                          /* len(block_out_channels): 4 (SD v1.5) / 3 (SDXL) */
  int block_out_channels[CFGPP_MAX_LEVELS];
  int down_has_attn[CFGPP_MAX_LEVELS];     /* CrossAttnDownBlock2D -> 1, DownBlock2D -> 0 */
  int up_has_attn[CFGPP_MAX_LEVELS];       /* in up_blocks order */
  int layers_per_block;                    /* 2 */
  int transformer_layers[CFGPP_MAX_LEVELS];/* per down level; mid uses the last; up uses reversed */
  int num_heads[CFGPP_MAX_LEVELS];         /* diffusers `attention_head_dim` (= number of heads) */
  int cross_attention_dim;                 /* 768 / 2048 */
  int use_linear_projection;               /* 0: 1x1-conv proj_in/out (SD v1.5), 1: Linear (SDXL) */
  int norm_num_groups;                     /* 32 */
  float norm_eps;                          /* 1e-5 (Transformer2DModel's GroupNorm uses 1e-6) */
  int addition_time_embed_dim;             /* 0: no add-embedding; 256: SDXL text_time */
  int projection_class_embeddings_input_dim; /* 2816 (SDXL base: 6 time ids), 2560 (SDXL refiner: 5) */
  int pooled_dim;                          /* 1280 */
  int prediction_type;                     /* 0: the UNet predicts epsilon; 1: v (SD 2.0-v / 2.1 at 768^2). Read by
                                              cfgpp_create_ex only; cfgpp_create takes the layout that ends at
                                              pooled_dim and means epsilon. */
} cfgpp_model_desc;

/* dtype codes */
#define CFGPP_F16 0
#define CFGPP_F32 1

/* sampler update fused behind the UNet (cfgpp_set_schedule `method`) */
#define CFGPP_STEP_NONE 0            /* no update: expose eps_uc / eps_c only */
#define CFGPP_STEP_DDIM_CFGPP 1      /* ddim_cfg++ (+_lightning)  latent_diffusion.py:660-666, latent_sdxl.py:738-744 */
#define CFGPP_STEP_DDIM_INV_CFGPP 2  /* inversion of ddim_inversion_cfg++  latent_diffusion.py:904-908 */
#define CFGPP_STEP_DPMPP2M_CFGPP 3   /* dpm++_2m_cfgpp  latent_sdxl.py:902-919 */
#define CFGPP_STEP_DDIM_CFG 4        /* plain-CFG ddim step and inversion step (baselines)  latent_diffusion.py:283-287 */

/* Per-step scalars, computed by the host exactly as the reference computes them (fp32 torch CPU ops). */
typedef struct cfgpp_step_coef {
  float lambda_;         /* cfg_guidance */
  float c0, c1, c2, c3;  /* DDIM: sqrt(1-a_t), sqrt(a_t), sqrt(a_next), sqrt(1-a_next)
                            DDIM-inv: sqrt(1-a_prev), sqrt(a_prev), sqrt(a_t), sqrt(1-a_t)
                            DPM++2M: c_out = -sigma_i, 1/sigma_i, sigma_{i+1}, unused */
  float d0, d1, d2, d3;  /* DPM++2M 2nd-order branch: -exp(-h), expm1(-h), 1/(2r), exp(-h) */
  int second_order;      /* VE-cast family bits: 1 = 2M update (else the Euler-CFG++ update: first step / sigma_next == 0 /
                            euler solvers), 2 = extrapolate with the guided estimate (plain-CFG euler, dpm++_2m),
                            4 = 2M difference term on the guided estimate (SD v1.5 dpm++_2m_cfg++),
                            8 = ancestral (euler_a, dpm++_2s_a: latent_diffusion.py:757-760, :823): after the update add
                                noise[slot c3] * d3 (sigma_up), the table comes from cfgpp_set_noise,
                            16 / 32 = the two UNet calls of a DPM-Solver++(2S) step (latent_diffusion.py:796-821), one
                                schedule entry each: 16 = midpoint, d0 = sigma_s / sigma_t, d1 = expm1(-h r) (x is parked,
                                the state becomes x_2); 32 = final, d0 = exp(-h), d1 = sigma_down / sigma_t,
                                d2 = expm1(-h) (plain-CFG form when bit 2 is set) */
} cfgpp_step_coef;

typedef struct cfgpp_step_state {
  float t;         /* timestep fed to the UNet (DDIM: t; DPM++: sigma_to_t(sigma_i) = t-1) */
  float in_scale;  /* model input scale c_in (1.0 for DDIM) */
  cfgpp_step_coef coef;
} cfgpp_step_state;

typedef struct cfgpp_handle cfgpp_handle;

int cfgpp_version(void);
const char* cfgpp_last_error(void);

/* ---- model lifetime: replaces pipe.unet obtained at latent_diffusion.py:67 / latent_sdxl.py:50,391 ---------- */
int cfgpp_create(const cfgpp_model_desc* desc, int device, cfgpp_handle** out);
/* desc_bytes = sizeof(cfgpp_model_desc), or offsetof(cfgpp_model_desc, prediction_type) for the layout without it (then
 * identical to cfgpp_create). */
int cfgpp_create_ex(const cfgpp_model_desc* desc, size_t desc_bytes, int device, cfgpp_handle** out);
int cfgpp_destroy(cfgpp_handle* h);
/* One call per state-dict entry under its diffusers key (SURVEY.md A.5), fp16 or fp32 device tensor. */
int cfgpp_load_weight(cfgpp_handle* h, const char* diffusers_key, const void* data_dev, const int64_t* shape, int ndim,
                      int dtype, void* stream);
/* Repack into kernel-native layouts (conv [Cout][9][Cin], fused QKV / KV, interleaved GEGLU, concatenated
 * time_emb_proj). Fails listing the first missing key if the state dict is incomplete. */
int cfgpp_finalize_weights(cfgpp_handle* h, void* stream);
/* Build the launch plan + workspace for `batch` images of latent size (h_lat, w_lat); UNet batch is 2*batch. */
int cfgpp_prepare(cfgpp_handle* h, int batch, int h_lat, int w_lat);
int cfgpp_workspace_bytes(cfgpp_handle* h, size_t* bytes);
/* Algorithmic FLOPs (2*MACs of conv/linear/QK^T/PV as the reference executes them) of one 2*batch UNet forward,
 * and the number of kernel launches one fused step enqueues. */
int cfgpp_forward_flops(cfgpp_handle* h, double* flops);
int cfgpp_launches_per_step(cfgpp_handle* h, int* n);
/* Accounting of the prepared plan, all per 2*batch UNet forward: step_flops = FLOPs the fused step EXECUTES every step
 * (excludes what runs once per prompt); prompt_flops / prompt_launches = the once-per-set_prompt part (cross-attention
 * K/V projections, SDXL add-embedding). cfgpp_forward_flops == step_flops + prompt_flops is the reference-equivalent
 * algorithmic figure (diffusers recomputes the K/V projections every step). */
int cfgpp_plan_stats(cfgpp_handle* h, double* step_flops, double* prompt_flops, int* prompt_launches);

/* ---- LoRA adapters: replaces diffusers' load_lora_weights + fuse_lora. For a weight W viewed as [N, K] (K = every
 * dimension after the first, a 3x3 conv in its (Cout,Cin,3,3) order) and adapters a with down_a [rank_a, K],
 * up_a [N, rank_a], alpha_a and a user scale s_a:
 *     W_eff = fp16( fp32(W) + sum_a c_a * sum_r up_a[n,r] down_a[r,k] ),   c_a = s_a * alpha_a / rank_a   (fp32)
 * with fp16 factors, fp32 accumulation and ONE rounding. W_eff is always formed from a pristine copy of W, written into
 * W's own device storage, and every kernel-native repack that reads W (conv layout, fused q|k|v and k|v, head padding,
 * GEGLU interleave, concatenated time_emb_proj, LayerNorm fold) is re-run into the buffer it already occupies: the
 * prepared plan and its captured graph stay as they are. ---------------------------------------------------------- */
/* After cfgpp_finalize_weights. adapter: id 0..63; down_dev / up_dev: device tensors of `dtype` (fp32 is rounded to fp16
 * once), copied; rank 1..128; at most 4 adapters per weight. The first adapter on a key takes that key's pristine
 * backup. Fails naming the key when it is missing, 1-D, or already targeted by this adapter. Merges nothing yet. */
int cfgpp_lora_add(cfgpp_handle* h, int adapter, const char* diffusers_weight_key, const void* down_dev,
                   const void* up_dev, int rank, float alpha, int dtype, void* stream);
/* Merges every targeted weight at scales_host[adapter id] (n_adapters = highest id + 1) and refreshes the packed copies,
 * all enqueued on `stream`. Afterwards cfgpp_run_steps / cfgpp_unet_forward fail until cfgpp_set_prompt is called again:
 * the cross-attention K/V and the add-embedding of the bound prompt came from the previous weights. */
int cfgpp_lora_set_scales(cfgpp_handle* h, const float* scales_host, int n_adapters, void* stream);
/* The base weights bit for bit; factors and backups are freed (synchronises `stream`). The prompt goes stale as above. */
int cfgpp_lora_clear(cfgpp_handle* h, void* stream);
/* backup_bytes: device memory held by pristine copies; bytes_moved: bytes the last set_scales / clear read and wrote
 * (merge and every refreshed packer), computed from shapes. Any pointer may be NULL. */
int cfgpp_lora_stats(cfgpp_handle* h, int* n_adapters, int* n_targets, size_t* backup_bytes, size_t* bytes_moved);

/* ---- per-prompt conditioning: the tensors predict_noise concatenates (latent_sdxl.py:178-182, 249-257) ------ */
/* ctx_dev: (2*batch, 77, cross_dim) fp16 = cat([uc, c]); pooled_dev: (add_rows, pooled_dim) fp16;
 * time_ids_dev: (add_rows, n_time_ids) fp32, n_time_ids = (projection_class_embeddings_input_dim - pooled_dim) /
 * addition_time_embed_dim (6 for the SDXL base, 5 for the SDXL refiner; 1..8, checked at create); add_rows is 2*batch, or batch when the reference does not duplicate the added
 * conditions (cfg_guidance in {0,1}: latent_sdxl.py:249-252 — rows then broadcast over both halves).
 * pooled/time_ids are ignored (may be NULL) for models without add-embedding. n_ctx = tokens per row (77). */
int cfgpp_set_prompt(cfgpp_handle* h, const void* ctx_dev, int n_ctx, const void* pooled_dev, const float* time_ids_dev,
                     int add_rows, void* stream);

/* ---- un-fused seam == predict_noise ------------------------------------------------------------------------- */
/* z_dev: (batch,4,h,w) NCHW of z_dtype; model input is z * in_scale; outputs (batch,4,h,w) fp16 each: the raw model
 * output, i.e. v for a prediction_type = 1 handle (cfgpp_op_v_to_eps converts it). */
int cfgpp_unet_forward(cfgpp_handle* h, const void* z_dev, int z_dtype, float t, float in_scale, void* eps_uc_dev,
                       void* eps_c_dev, void* stream);

/* Profiling aid: the same un-fused forward with a CUDA-event pair around every plan entry. Arrays are caller-owned
 * host buffers of max_n entries; kind: 0 linear GEMM, 1 conv3x3, 2 attention, 3 other; names_host holds max_n
 * NUL-terminated strings of name_stride bytes each (may be NULL). Synchronises the stream (not a hot-path call). */
int cfgpp_profile_forward(cfgpp_handle* h, const void* z_dev, int z_dtype, float t, float in_scale, int max_n,
                          int* n_out, float* ms_host, double* flops_host, int* kind_host, char* names_host,
                          int name_stride, void* stream);

/* ---- fused trajectory: UNet + CFG++ mix + scheduler update per step, one CUDA graph replayed per step -------- */
int cfgpp_set_schedule(cfgpp_handle* h, int method, int state_dtype, const cfgpp_step_state* steps_host, int nsteps,
                       void* stream);
/* Copy the caller's initial state into the library's state buffer (z: zT / x0; aux: old_denoised or NULL). */
int cfgpp_set_state(cfgpp_handle* h, const void* z_dev, int z_dtype, void* stream);
/* Ancestral samplers: the trajectory's fresh noise, drawn up front in the order the reference's loop would draw it
 * (`torch.randn_like(x)` once per step with sigma_next > 0). noise_dev: fp16 [slots][batch,4,h,w]; copied. */
int cfgpp_set_noise(cfgpp_handle* h, const void* noise_dev, int slots, void* stream);
/* Per-image guidance: lambda_host is a host array of n = batch fp32 values (copied; the caller may reuse it on
 * return). While it is set, the guidance mix of every step (fused cfgpp_run_steps and un-fused cfgpp_apply_step, every
 * method and second_order bit) uses lambda[b] for image b instead of cfgpp_step_coef.lambda_, with the same rounding.
 * n = 0 clears it; cfgpp_prepare clears it too. Enqueued on `stream`; a captured trajectory graph stays valid. */
int cfgpp_set_guidance(cfgpp_handle* h, const float* lambda_host, int n, void* stream);
/* v-prediction handles (prediction_type = 1): ab_host holds nsteps (a, b) pairs, one per entry of the current schedule,
 * a = sqrt(abar), b = sqrt(1 - abar) of the noise level that entry's update assigns to the state the UNet sees (DDIM
 * modes: a = c1, b = c0; STEP_DPMPP2M_CFGPP: a = in_scale, b = sigma * in_scale). Each fused step converts the conv
 * output v to eps = fp16(fp32(a v) + fp32(b x_in)), x_in the UNet input, before the guidance mix. Required after every
 * cfgpp_set_schedule of such a handle before cfgpp_run_steps; refused by epsilon handles. */
int cfgpp_set_v_coefs(cfgpp_handle* h, const float* ab_host, int nsteps, void* stream);
/* Run `nsteps` consecutive steps starting at schedule index `first_step` on the internal state. */
int cfgpp_run_steps(cfgpp_handle* h, int first_step, int nsteps, void* stream);
/* which: 0 = state z (same dtype as the state), 1 = z0t of the last executed step. */
int cfgpp_get_state(cfgpp_handle* h, int which, void* out_dev, void* stream);
/* Standalone update from caller-provided eps (callback path: the caller may have modified nothing, it just needs
 * z0t / zt materialised between UNet calls). Applies schedule entry `step` to the internal state. Takes eps for every
 * prediction_type (a v model's caller converts first, cfgpp_op_v_to_eps). */
int cfgpp_apply_step(cfgpp_handle* h, int step, const void* eps_uc_dev, const void* eps_c_dev, void* stream);

/* ---- ControlNet (diffusers ControlNetModel, guess_mode off): spatial conditioning of a UNet handle ---------------
 * A ControlNet handle holds its own weights under the ControlNetModel keys (`conv_in.*`, `time_embedding.*`,
 * `add_embedding.*`, `down_blocks.*`, `mid_block.*`, `controlnet_cond_embedding.*`, `controlnet_down_blocks.{k}.*`,
 * `controlnet_mid_block.*`), loaded with cfgpp_load_weight / cfgpp_finalize_weights and destroyed with cfgpp_destroy.
 * It is run through the UNet handle it is attached to. Per UNet call, on the full 2*batch rows:
 *   sample  = fp16(fp16(conv_in(z * in_scale)) + cond),  cond = controlnet_cond_embedding(fp16(image)) (batch rows,
 *             shared by both CFG halves), then the ControlNet's own time / add-embedding, down blocks and mid block
 *             on the UNet's timestep, context and added conditions;
 *   r_k     = fp16(zero_conv_k(res_k) + bias_k) for every down-path skip tensor k and the mid-block output;
 *   skip_k' = fp16(float(skip_k) + float(fp16(float(r_k) * s))), the same for the UNet's mid-block output, with s the
 *             conditioning scale of the step. The UNet's down path and mid block see the un-added tensors; only the up
 *             path sees the sums. */
typedef struct cfgpp_controlnet_desc {
  cfgpp_model_desc model;       /* down / mid geometry of the ControlNet (up_* fields ignored; out_channels 4) */
  int conditioning_channels;    /* 3 (RGB) */
  int num_embedding_levels;     /* len(conditioning_embedding_out_channels): 4 (the embedding downsamples by 8) */
  int embedding_channels[CFGPP_MAX_LEVELS]; /* (16, 32, 96, 256) */
} cfgpp_controlnet_desc;
int cfgpp_controlnet_create(const cfgpp_controlnet_desc* desc, int device, cfgpp_handle** out);
/* On a ControlNet handle, every entry point that prepares, conditions, runs or schedules a UNet (cfgpp_prepare,
 * cfgpp_set_prompt, cfgpp_unet_forward, cfgpp_profile_forward, cfgpp_set_schedule .. cfgpp_apply_step, cfgpp_lora_*,
 * cfgpp_attach_controlnet's first argument, cfgpp_set_control_*) fails with an error status. cfgpp_workspace_bytes of a
 * UNet handle counts the attached ControlNet's workspace too. */
/* Attach a finalized ControlNet handle to a UNet handle (cn = NULL detaches). num_levels, block_out_channels,
 * layers_per_block, cross_attention_dim and the add-embedding dims must equal the UNet's (the error names the first
 * field that differs). Attaching or detaching drops the prepared plan: the next cfgpp_prepare builds one plan of
 * ControlNet prologue, ControlNet down + mid, UNet down + mid, zero convs (in place into the UNet's skip tensors and
 * mid output), UNet up path; cfgpp_run_steps, cfgpp_unet_forward and cfgpp_profile_forward all run it.
 * cfgpp_set_prompt also projects the ControlNet's cross-attention K/V and its add-embedding. A ControlNet is attached
 * to at most one UNet at a time and must outlive the attachment (destroying either end detaches). */
int cfgpp_attach_controlnet(cfgpp_handle* h, cfgpp_handle* cn);
/* image_dev: (batch, 3, 8*h_lat, 8*w_lat) NCHW RGB in [0, 1] of `dtype`, for the prepared shape. Runs the conditioning
 * embedding once into the plan's buffer; cfgpp_run_steps / cfgpp_unet_forward of an attached handle fail until it has
 * been called after the last cfgpp_prepare. */
int cfgpp_set_control_image(cfgpp_handle* h, const void* image_dev, int dtype, void* stream);
/* The conditioning scale s of cfgpp_unet_forward and of every step (1.0 after create); clears the per-entry table
 * (enqueued on `stream`). */
int cfgpp_set_control_scale(cfgpp_handle* h, float scale, void* stream);
/* One scale per entry of the current schedule (host [nsteps], copied), read on the device by the step selection:
 * changing it never recaptures the step graph. cfgpp_set_schedule and cfgpp_set_control_scale clear it. */
int cfgpp_set_control_scales(cfgpp_handle* h, const float* scales_host, int nsteps, void* stream);
/* The conditioning embedding on its own, on a ControlNet handle: image (batch, 3, height, width) as above ->
 * out_dev (batch, height/8, width/8, C0) NHWC fp16. */
int cfgpp_controlnet_embed(cfgpp_handle* cn, const void* image_dev, int dtype, int batch, int height, int width,
                           void* out_dev, void* stream);

/* ---- IP-Adapter (Ye et al. 2023; diffusers ImageProjection + IPAdapterAttnProcessor2_0): a reference image as a
 * prompt, on a UNet handle. Weights, under diffusers' UNet-side keys:
 *   image_proj.proj.{weight,bias}  [n_tokens * D, E], [n_tokens * D]   (D = cross_attention_dim, E = image embed width)
 *   image_proj.norm.{weight,bias}  [D]
 *   {block}.attn2.processor.to_k_ip.0.weight, {block}.attn2.processor.to_v_ip.0.weight  [C, D] for every cross-attention
 *   block of the UNet ({block} = e.g. down_blocks.1.attentions.0.transformer_blocks.0; the original checkpoints'
 *   `ip_adapter.{i}` index maps to it in diffusers' attn_processors order, cfgpp_b200/ip_adapter.py).
 * Per UNet call, with tokens = LayerNorm_D(rows of fp16(embeds W_proj^T + b_proj)) [2*batch * n_tokens, D] projected
 * once per image (K2 = tokens W_k_ip^T, V2 = tokens W_v_ip^T, fp16), every attn2 computes
 *   out = fp16(O_txt / l_txt + s * O_ip / l_ip)
 * in one kernel: the text softmax attention and the image softmax attention (each with its own max and sum) summed in
 * fp32 and rounded once (diffusers rounds each term to fp16 first), then to_out as before. s = 0 gives the plain
 * cross-attention bit for bit. An attached ControlNet sees the text context only. -------------------------------- */
/* After cfgpp_finalize_weights, any number of times (a key loaded again replaces its tensor); fails naming a key that
 * is not one of the above, has no cross-attention block, or whose shape differs from the block's to_k. Loading drops
 * the image projection (call cfgpp_set_ip_image_embeds again); loading a key a second time also drops the prepared
 * plan. The UNet's own weights are untouched. */
int cfgpp_ip_adapter_load_weight(cfgpp_handle* h, const char* key, const void* data_dev, const int64_t* shape, int ndim,
                                 int dtype, void* stream);
/* Attach the loaded adapter (n_tokens 1..64, image_embed_dim E a multiple of 8) or detach it (cfgpp_ip_adapter_clear;
 * its weights stay loaded). Either drops the prepared plan: the next cfgpp_prepare builds every attn2 with or without
 * the image segment; without an adapter the plan is exactly the one built before any adapter was attached. */
int cfgpp_ip_adapter_attach(cfgpp_handle* h, int n_tokens, int image_embed_dim);
int cfgpp_ip_adapter_clear(cfgpp_handle* h);
/* embeds_dev: (2*batch, E) fp16 device tensor, rows in cfgpp_set_prompt's order (the unconditional half: zeros, as
 * diffusers' negative image embeds). Runs the image projection and every block's K2 / V2 projection now, into the
 * plan's buffers; cfgpp_run_steps / cfgpp_unet_forward of a handle with an adapter fail until it has been called after
 * the last cfgpp_prepare or weight load. */
int cfgpp_set_ip_image_embeds(cfgpp_handle* h, const void* embeds_dev, void* stream);
/* The scale s (1.0 after create): one fp32 device word every decoupled cross-attention launch reads, written on
 * `stream`; never recaptures the step graph. */
int cfgpp_set_ip_adapter_scale(cfgpp_handle* h, float scale, void* stream);
/* ---- IP-Adapter Plus (diffusers IPAdapterPlusImageProjection, the Perceiver "Resampler"): the image tokens come from
 * the image encoder's penultimate hidden states h [2*batch, seq_len, E] instead of one pooled embedding. Weights, loaded
 * with cfgpp_ip_adapter_load_weight under the original checkpoint's `image_proj.*` keys (inner = 64 * heads,
 * F = ff_mult * dim, D = cross_attention_dim):
 *   image_proj.latents [1, Q, dim]; proj_in.{weight,bias} [dim, E], [dim]; proj_out.{weight,bias} [D, dim], [D];
 *   norm_out.{weight,bias} [D]; per layer i: layers.{i}.0.norm1 (on x) / .norm2 (on the latents) {weight,bias} [dim],
 *   layers.{i}.0.to_q.weight [inner, dim], layers.{i}.0.to_kv.weight [2 * inner, dim] (k rows first, then v),
 *   layers.{i}.0.to_out.weight [dim, inner], layers.{i}.1.0.{weight,bias} [dim], layers.{i}.1.1.weight [F, dim],
 *   layers.{i}.1.3.weight [dim, F]
 * plus the per-block to_k_ip / to_v_ip above. Each Linear rounds once to fp16, every LayerNorm has eps 1e-5:
 *   x = proj_in(h); lat = latents (per image)
 *   per layer: kv = [LN0(x), LN1(lat)] (seq_len + Q rows), lat = to_out(SDPA(to_q(LN1(lat)), to_k(kv), to_v(kv))) + lat
 *              (heads of 64, scale 1/8, no bias), lat = W2 gelu_erf(W1 LN_ff(lat)) + lat (bias-free)
 *   tokens = norm_out(proj_out(lat))  [2*batch * Q, D]
 * and the tokens feed every attn2 as the plain adapter's do. */
typedef struct cfgpp_ip_resampler_desc {
  int num_queries; /* Q, the image tokens: 1..64 (the Plus checkpoints: 16) */
  int embed_dim;   /* E, the hidden-state width: a multiple of 64 (ViT-H/14: 1280) */
  int seq_len;     /* rows of h per image (ViT-H/14 at 224: 257) */
  int dim;         /* the Resampler's width: a multiple of 64, <= 2048 (SD v1.5 Plus: 768, SDXL Plus: 1280) */
  int heads;       /* heads of 64 (12 / 20) */
  int depth;       /* layers (4) */
  int ff_mult;     /* feed-forward width / dim (4) */
} cfgpp_ip_resampler_desc;
/* Attach the loaded Plus adapter: like cfgpp_ip_adapter_attach (which, like cfgpp_ip_adapter_clear, also detaches a
 * Resampler), and fails naming a key above that is missing or whose shape does not fit `desc`. */
int cfgpp_ip_adapter_attach_resampler(cfgpp_handle* h, const cfgpp_ip_resampler_desc* desc);
/* hidden_dev: (2*batch, seq_len, E) fp16 device tensor, rows in cfgpp_set_prompt's order (the unconditional half: the
 * encoder's hidden states of an all-zero preprocessed image, as diffusers). Runs the Resampler and every block's K2 / V2
 * projection now; the counterpart of cfgpp_set_ip_image_embeds, which refuses a Resampler (and this one, a plain
 * adapter). */
int cfgpp_set_ip_image_hidden_states(cfgpp_handle* h, const void* hidden_dev, void* stream);

/* ---- T2I-Adapter (Mou et al. 2023; diffusers T2IAdapter, `full_adapter` / `full_adapter_xl`): spatial conditioning by
 * four feature maps computed once per image and added into a UNet handle's down path at every step. An adapter handle
 * holds the weights under diffusers' keys (`adapter.conv_in.*`, `adapter.body.{i}.in_conv.*`,
 * `adapter.body.{i}.resnets.{j}.block1.*` (3x3), `adapter.body.{i}.resnets.{j}.block2.*` (1x1)) and runs, on an image
 * x (batch, in_channels, H, W) in [0, 1], in fp16:
 *   x = conv_in(pixel_unshuffle(fp16(x), downscale_factor))       (channel c*f*f + i*f + j holds pixel (f*y+i, f*x+j))
 *   per block i: [x = avgpool2x2(x) if down] [x = in_conv(x) if cin != cout]
 *                num_res_blocks x { x = fp16(fp16(block2(relu(block1(x)))) + x) };  feature_i = fp16(x * scale)
 * full (SD):     blocks (c0,c0), (c0,c1,down), (c1,c2,down), (c2,c3,down): features at /f, /2f, /4f, /8f;
 * full_xl (SDXL): blocks (c0,c0), (c0,c1), (c1,c2,down), (c3,c3) with c2 == c3: features at /f, /f, /2f, /2f.
 * H and W must be multiples of the total factor (8f for full, 2f for full_xl): the average pool never pads. */
typedef struct cfgpp_t2i_adapter_desc {
  int kind;              /* 0: full_adapter (SD v1.5 / SD 2.x), 1: full_adapter_xl (SDXL) */
  int in_channels;       /* 1 (sketch, canny) or 3 (RGB) */
  int channels[4];       /* (320, 640, 1280, 1280) */
  int num_res_blocks;    /* 2 */
  int downscale_factor;  /* 8 (full) or 16 (full_xl) */
} cfgpp_t2i_adapter_desc;
typedef struct cfgpp_t2i_adapter_handle cfgpp_t2i_adapter_handle;
int cfgpp_t2i_adapter_create(const cfgpp_t2i_adapter_desc* desc, int device, cfgpp_t2i_adapter_handle** out);
int cfgpp_t2i_adapter_destroy(cfgpp_t2i_adapter_handle* ad);
int cfgpp_t2i_adapter_load_weight(cfgpp_t2i_adapter_handle* ad, const char* key, const void* data_dev,
                                  const int64_t* shape, int ndim, int dtype, void* stream);
/* Checks every weight's exact shape (the error names the first missing or mis-shaped key) and packs the 3x3 convs. */
int cfgpp_t2i_adapter_finalize_weights(cfgpp_t2i_adapter_handle* ad, void* stream);
/* image_dev: (batch, in_channels, H, W) NCHW of `dtype` (fp16 / fp32), batch 1..8. features_out[k]: device buffers for
 * feature k, NHWC fp16 (batch, h_k, w_k, channels_k), written already multiplied by `scale`. The launch plan is built
 * for (batch, H, W) at the first call and kept until another shape arrives. */
int cfgpp_t2i_adapter_forward(cfgpp_t2i_adapter_handle* ad, const void* image_dev, int dtype, int batch, int H, int W,
                              float scale, void* const* features_out, void* stream);
/* FLOPs of the prepared forward and its workspace bytes (0 before the first forward). */
int cfgpp_t2i_adapter_stats(cfgpp_t2i_adapter_handle* ad, double* flops, size_t* workspace_bytes);
/* On a UNet handle: expect n_features T2I-Adapter features (0 detaches). Either drops the prepared plan. The next
 * cfgpp_prepare places feature k, in order, on (diffusers' down_intrablock_additional_residuals):
 *   a CrossAttnDownBlock2D: the output of its last (resnet, attention) pair, before its downsampler (so the skip
 *   tensor and the downsampler's input are the sum); a DownBlock2D: its output, after its downsampler if it has one;
 *   a feature left after the down blocks: the mid-block output.
 * It fails unless n_features is num_levels or num_levels + 1 (the last down block has no downsampler, so the mid-block
 * output always has the last down placement's shape). Each placement is one launch in the step graph: rows r of h [2*batch, HW, C] become
 *   h = fp16(float(h) + float(feature[r mod batch]))
 * when the step's T2I word is on, and are left untouched (no write) when it is off. The adds come before an attached
 * ControlNet's residuals; the ControlNet's own down path gets no features. */
int cfgpp_t2i_attach(cfgpp_handle* h, int n_features);
/* features_dev[k]: (batch, h_k, w_k, C_k) NHWC fp16 for the prepared shape, copied into the plan's buffers (both CFG
 * halves read the same rows). cfgpp_run_steps / cfgpp_unet_forward of a handle with features attached fail until it
 * has been called after the last cfgpp_prepare. */
int cfgpp_set_t2i_features(cfgpp_handle* h, const void* const* features_dev, void* stream);
/* The T2I word of cfgpp_unet_forward and of every entry of a new schedule (on = 1 after create); clears the per-entry
 * table (enqueued on `stream`). */
int cfgpp_set_t2i_active(cfgpp_handle* h, int on, void* stream);
/* One word per entry of the current schedule (host [nsteps], nonzero = on), read on the device by the step selection:
 * diffusers' `i < int(num_inference_steps * adapter_conditioning_factor)`. cfgpp_set_schedule and cfgpp_set_t2i_active
 * clear it. */
int cfgpp_set_t2i_steps(cfgpp_handle* h, const int* on_host, int nsteps, void* stream);

/* ---- AutoencoderKL decoder (SURVEY.md section 8 f2): replaces `self.vae.decode(zt / scaling_factor).sample` of
 * latent_sdxl.py:155-164 (VAE madebyollin/sdxl-vae-fp16-fix, :44) and latent_diffusion.py:123-129 on the same conv /
 * GEMM / GroupNorm kernels. Weights under the diffusers AutoencoderKL keys (`post_quant_conv.*`, `decoder.*`). ----- */
typedef struct cfgpp_vae_desc {
  int latent_channels;                       /* 4 */
  int out_channels;                          /* 3 */
  int num_levels;                            /* len(block_out_channels): 4 */
  int block_out_channels[CFGPP_MAX_LEVELS];  /* (128, 256, 512, 512) */
  int layers_per_block;                      /* 2 (the decoder's up blocks hold layers_per_block + 1 resnets) */
  int norm_num_groups;                       /* 32 */
  float scaling_factor;                      /* 0.13025 (SDXL) / 0.18215 (SD v1.5) */
} cfgpp_vae_desc;
typedef struct cfgpp_vae_handle cfgpp_vae_handle;
int cfgpp_vae_create(const cfgpp_vae_desc* desc, int device, cfgpp_vae_handle** out);
int cfgpp_vae_destroy(cfgpp_vae_handle* h);
int cfgpp_vae_load_weight(cfgpp_vae_handle* h, const char* diffusers_key, const void* data_dev, const int64_t* shape,
                          int ndim, int dtype, void* stream);
int cfgpp_vae_finalize_weights(cfgpp_vae_handle* h, void* stream);
/* zt_dev: (batch,4,h,w) NCHW of z_dtype — the SCALED latent the samplers return (the division by scaling_factor
 * happens inside, in zt's dtype, as in the reference); image_dev: (batch,3,8h,8w) NCHW fp16 (num_levels = 4).
 * The plan / workspace for (batch,h,w) is built on first use and cached. */
int cfgpp_vae_decode(cfgpp_vae_handle* h, const void* zt_dev, int z_dtype, int batch, int h_lat, int w_lat,
                     void* image_dev, void* stream);
/* ENCODER half — replaces `self.vae.encode(x).latent_dist.sample() * scaling_factor` (latent_sdxl.py:151-152,
 * latent_diffusion.py:117-121), the front end of the inversion / editing solvers. Needs the `encoder.*` and
 * `quant_conv.*` weights to have been loaded. image_dev: (batch,3,H,W) NCHW of image_dtype in [-1, 1];
 * noise_dev: (batch,4,H/8,W/8) fp16 — the `randn` draw of DiagonalGaussianDistribution.sample, made by the caller —
 * or NULL for the posterior mean; latent_out: (batch,4,H/8,W/8) fp32 (the fp16 module's output under the reference's
 * autocast: `exp` promotes the posterior's std to fp32), already multiplied by scaling_factor. */
int cfgpp_vae_encode(cfgpp_vae_handle* h, const void* image_dev, int image_dtype, int batch, int height, int width,
                     const void* noise_dev, void* latent_out, void* stream);
/* Algorithmic FLOPs of one decode of the prepared shape, and its activation workspace. */
int cfgpp_vae_stats(cfgpp_vae_handle* h, double* flops, size_t* workspace_bytes);

/* ---- CLIP text encoder (SURVEY.md section 8 f3): replaces `self.text_encoder(ids)[0]` of latent_diffusion.py:93-115 and
 * `text_enc(ids, output_hidden_states=True)` -> `hidden_states[-2]` / `[-(clip_skip + 2)]` / `[0]` of
 * latent_sdxl.py:77-93 (transformers CLIPTextModel: openai/clip-vit-large-patch14; CLIPTextModelWithProjection:
 * OpenCLIP ViT-bigG). Weights under the transformers keys (`text_model.*`, `text_projection.weight`). Tokenisation
 * stays on the host (cfgpp_b200/tokenizer.py). ----- */
typedef struct cfgpp_clip_desc {
  int vocab_size;        /* 49408 */
  int max_positions;     /* 77 */
  int hidden_size;       /* 768 (CLIP-L) / 1280 (bigG); heads are 64 wide */
  int intermediate_size; /* 3072 / 5120 */
  int num_layers;        /* 12 / 32 */
  int num_heads;         /* 12 / 20 */
  int hidden_act;        /* 0 = quick_gelu (CLIP-L), 1 = gelu (bigG) */
  int projection_dim;    /* 0 = CLIPTextModel; > 0 = CLIPTextModelWithProjection (1280) */
  float layer_norm_eps;  /* 1e-5 */
} cfgpp_clip_desc;
typedef struct cfgpp_clip_handle cfgpp_clip_handle;
int cfgpp_clip_create(const cfgpp_clip_desc* desc, int device, cfgpp_clip_handle** out);
int cfgpp_clip_destroy(cfgpp_clip_handle* h);
int cfgpp_clip_load_weight(cfgpp_clip_handle* h, const char* transformers_key, const void* data_dev, const int64_t* shape,
                           int ndim, int dtype, void* stream);
int cfgpp_clip_finalize_weights(cfgpp_clip_handle* h, void* stream);
/* input_ids_dev: (batch, n_tokens) int32 token ids; pooled_index_dev: (batch) int32 row of the pooled token (the
 * <|endoftext|> position the model's eos rule selects; may be null when pooled_out is null). Outputs, fp16, each may
 * be null: hidden_out (batch, n_tokens, hidden) = hidden_states[num_layers - skip] (skip = 1: the penultimate layer SDXL
 * conditions on; skip = clip_skip + 1 in general); last_hidden_out = final_layer_norm(hidden_states[-1]) (what SD v1.5
 * conditions on); pooled_out (batch, projection_dim or hidden) = text_embeds / pooler_output. */
int cfgpp_clip_encode(cfgpp_clip_handle* h, const int32_t* input_ids_dev, const int32_t* pooled_index_dev, int batch,
                      int n_tokens, int skip, void* hidden_out, void* last_hidden_out, void* pooled_out, void* stream);
int cfgpp_clip_stats(cfgpp_clip_handle* h, double* flops, size_t* workspace_bytes);

/* ---- CLIP vision tower: transformers CLIPVisionModelWithProjection (IP-Adapter's image encoder: ViT-H/14 for SD v1.5,
 * ViT-bigG/14 for SDXL). Weights under its keys (`vision_model.*`, `visual_projection.weight`). The patch conv runs as
 * an unfold and a GEMM, the layers are the text towers' pre-LN loop with non-causal flash attention (heads zero-padded
 * to a multiple of 64 columns), then post_layernorm of the CLS row and visual_projection. ----- */
typedef struct cfgpp_clip_vision_desc {
  int hidden_size;       /* 1280 (ViT-H) / 1664 (bigG) */
  int intermediate_size; /* 5120 / 8192 */
  int num_layers;        /* 32 / 48 */
  int num_heads;         /* 16 (heads of 80 / 104) */
  int image_size;        /* 224 */
  int patch_size;        /* 14 */
  int hidden_act;        /* 0 = quick_gelu, 1 = gelu */
  int projection_dim;    /* 1024 / 1280 */
  float layer_norm_eps;  /* 1e-5 */
} cfgpp_clip_vision_desc;
typedef struct cfgpp_clip_vision_handle cfgpp_clip_vision_handle;
int cfgpp_clip_vision_create(const cfgpp_clip_vision_desc* desc, int device, cfgpp_clip_vision_handle** out);
int cfgpp_clip_vision_destroy(cfgpp_clip_vision_handle* h);
int cfgpp_clip_vision_load_weight(cfgpp_clip_vision_handle* h, const char* transformers_key, const void* data_dev,
                                  const int64_t* shape, int ndim, int dtype, void* stream);
int cfgpp_clip_vision_finalize_weights(cfgpp_clip_vision_handle* h, void* stream);
/* pixel_values_dev: (batch 1..16, 3, image_size, image_size) NCHW of `dtype`, CLIPImageProcessor's output (rounded to
 * fp16 as the fp16 model's conv input); image_embeds_out: (batch, projection_dim) fp16. */
int cfgpp_clip_vision_encode(cfgpp_clip_vision_handle* h, const void* pixel_values_dev, int dtype, int batch,
                             void* image_embeds_out, void* stream);
/* The same images -> hidden_out (batch, T, hidden_size) fp16 = hidden_states[num_layers - skip] (T = (image_size /
 * patch_size)^2 + 1; skip = 1: the penultimate layer IP-Adapter Plus reads; skip = num_layers: pre_layrnorm's output).
 * No post_layernorm, no projection; the layers after the wanted one do not run. */
int cfgpp_clip_vision_encode_hidden(cfgpp_clip_vision_handle* h, const void* pixel_values_dev, int dtype, int batch,
                                    int skip, void* hidden_out, void* stream);
int cfgpp_clip_vision_stats(cfgpp_clip_vision_handle* h, double* flops, size_t* workspace_bytes);

/* ---- operator-level entry points (one kernel each; used by the kernel parity tests and micro-benchmarks) ----- */
/* force_streamk (also in cfgpp_op_linear_lnfold): take the stream-K remainder split whenever its pieces are at least 2
 * k-blocks deep. The linear layers never take it otherwise; this lets tests reach the split's fix-up path. */
int cfgpp_op_linear(const void* a, int lda, const void* a2, int lda2, int k_split, const void* w, int M, int N, int K,
                    const void* bias, const void* addend, int ld_add, int add_rows_per_group, void* out, int ldc,
                    int geglu, int force_bn, int force_streamk, void* stream);
/* The LayerNorm-fold variants of cfgpp_op_linear (a [M,K], single source), exactly one of:
 *  stats_out (producer): besides out, writes per-row partial (sum, sum of squares) of the fp16 output as
 *    [2 * ceil(N / force_bn)][M] float2 — part 2 j + h covers columns [j BN + h BN / 2, j BN + (h + 1) BN / 2) of N
 *    block j; force_bn is required. out may alias addend (in-place residual add).
 *  stats_in (consumer): w is the folded weight of cfgpp_op_fold_ln, the epilogue applies
 *    rstd * acc - rstd * mean * ln_s[n] + ln_t[n] with mean / rstd over C = K from the first ln_parts parts of
 *    stats_in ([ln_parts][M] float2); bias and addend must be null (the bias is inside ln_t). */
int cfgpp_op_linear_lnfold(const void* a, const void* w, int M, int N, int K, const void* bias, const void* addend,
                           int ld_add, int add_rows_per_group, void* out, int ldc, int geglu, int force_bn,
                           int force_streamk, float* stats_out, const float* stats_in, int ln_parts, float ln_eps,
                           const float* ln_s, const float* ln_t, void* stream);
/* LayerNorm fold of w [N,K] fp16 with LayerNorm(K) gamma / beta (fp16) and an optional bias [N]: wf = fp16(w * gamma)
 * [N,K] fp16, s[n] = sum_k wf[n,k], t[n] = sum_k beta[k] w[n,k] + bias[n] (fp32). */
int cfgpp_op_fold_ln(const void* w, const void* gamma, const void* beta, const void* bias, void* wf, float* s, float* t,
                     int N, int K, void* stream);
/* The LoRA merge kernel on its own: out [N,K] fp16 = fp16(fp32(base) + sum_a coefs_host[a] * up_a down_a), downs[a]
 * [ranks[a], K] and ups[a] [N, ranks[a]] fp16 device tensors (host arrays of device pointers), ranks 1..128,
 * n_adapters 0..4, any N and K. out may be base. */
int cfgpp_op_lora_merge(const void* base, const void* const* downs, const void* const* ups, const int* ranks,
                        const float* coefs_host, int n_adapters, int N, int K, void* out, void* stream);
int cfgpp_op_conv3x3(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias,
                     const void* addend, int ld_add, int add_rows_per_group, void* out, int force_bn, void* stream);
/* Downsample2D: 3x3, stride 2 on NHWC x [B,H,W,Cin] (even H, W) -> [B,H/2,W/2,Cout]; the A tile is fetched by TMA with
 * element strides 2 (no im2col copy). pad = 1: the UNet's (symmetric zero padding); pad = 0: the AutoencoderKL encoder's
 * (one zero row / column AFTER the image, F.pad(x, (0, 1, 0, 1)) + un-padded convolution). */
int cfgpp_op_conv3x3_s2(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias, int pad,
                        void* out, void* stream);
/* The implicit-GEMM 3x3 convolution in all its modes: stride 1 / pad 1, stride 2 / pad 1, stride 2 / pad 0 (as above),
 * with the optional addend of cfgpp_op_conv3x3. The A tile comes through the tiled TMA box where the output geometry
 * allows it and through the im2col tensor map otherwise (any H, W); force_im2col != 0 takes the im2col map for every
 * geometry (both modes compute bit-identical results: same tile, same k order). */
int cfgpp_op_conv3x3_ex(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias,
                        const void* addend, int ld_add, int add_rows_per_group, void* out, int force_bn, int stride,
                        int pad, int force_im2col, void* stream);
/* The ControlNet zero-conv epilogue: out [M,N] = fp16(float(addend) + float(fp16(float(fp16(a w^T + bias)) * s))),
 * a [M,K], w [N,K], addend [M,N] fp16 (ld = N), s = *scale_dev (fp32, device). out may be addend (in place).
 * scale_dev = NULL is the plain residual epilogue of cfgpp_op_linear. */
int cfgpp_op_linear_scaled_residual(const void* a, const void* w, int M, int N, int K, const void* bias,
                                    const void* addend, const float* scale_dev, void* out, int force_bn, void* stream);
/* cfgpp_op_conv_in with an addend [B,H,W,Cout] NHWC fp16 shared by the `reps` repetitions:
 * out = fp16(fp16(conv_in(z)) + addend). */
int cfgpp_op_conv_in_add(const void* z, int z_dtype, const float* in_scale_dev, const void* w, const void* bias,
                         const void* addend, void* out, int B, int H, int W, int Cout, int reps, void* stream);
/* head h of q / k / v / out occupies columns [h*P, h*P + head_dim) with P = head_dim rounded up to a multiple of 64
 * (columns head_dim..P-1 must be zero in q / k / v and come back zero in out). */
int cfgpp_op_attention(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo, int B,
                       int H, int Nq, int Nkv, int head_dim, void* stream);
/* Decoupled cross-attention (IP-Adapter): cfgpp_op_attention over (k, v) plus a second segment of Nkv2 = 1..64 image
 * tokens k2 / v2 [B, Nkv2, H*P] (row strides ldk2 / ldv2) with a softmax of its own:
 *   out = fp16(O1 / l1 + s * O2 / l2),  s = *ip_scale_dev (fp32, device, read by the kernel),
 * summed in fp32 and rounded once, where diffusers rounds each term to fp16 first. s = 0 returns cfgpp_op_attention's
 * output bit for bit. */
int cfgpp_op_attention_ip(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, const void* k2,
                          int ldk2, const void* v2, int ldv2, int Nkv2, const float* ip_scale_dev, void* out, int ldo,
                          int B, int H, int Nq, int Nkv, int head_dim, void* stream);
int cfgpp_op_groupnorm(const void* x1, int C1, const void* x2, int C2, int B, int HW, const void* gamma,
                       const void* beta, float eps, int silu, void* out, void* stream);
int cfgpp_op_layernorm(const void* x, int M, int C, const void* gamma, const void* beta, float eps, void* out,
                       void* stream);
/* The two LayerNorms of an IP-Adapter Plus Resampler layer in one launch (C % 8 == 0, C <= 2048):
 * kv [NB, T + Q, C]: rows (b, 0..T-1) = LN(x[b]; g0, b0), rows (b, T..T+Q-1) = LN(lat[b]; g1, b1), x [NB, T, C],
 * lat [NB, Q, C]; q [NB, Q, C] = LN(lat; g1, b1) again. Every row equals cfgpp_op_layernorm's output for it, bit for bit. */
int cfgpp_op_ip_ln_concat(const void* x, const void* lat, int NB, int T, int Q, int C, const void* g0, const void* b0,
                          const void* g1, const void* b1, float eps, void* kv, void* q, void* stream);
/* noise_dev (may be null): fp16 ancestral-noise table [slots][n]; the slot is coef_host->c3 (second_order bit 8).
 * lambda_dev (may be null): a per-image guidance table fp32 [batch] (device); element i of the n belongs to image
 * i / (n / batch) and mixes with lambda_dev[image]. NULL uses coef_host->lambda_ (batch is then ignored). */
int cfgpp_op_cfgpp_step(const void* eps_uc, const void* eps_c, int n, int method, int state_dtype,
                        const cfgpp_step_coef* coef_host, void* z, void* aux, void* z0t_out, const void* noise_dev,
                        const float* lambda_dev, int batch, void* stream);
/* Sinusoidal embedding (diffusers get_timestep_embedding, flip_sin_to_cos): value i = vals_dev[i * val_stride] (fp32)
 * -> out[i * ld + col_off + (0 .. dim/2)] = cos, [.. + dim/2 .. dim) = sin, fp16; other columns are not written. */
int cfgpp_op_timestep_embedding(const float* vals_dev, int val_stride, int n, int dim, void* out, int ld, int col_off,
                                void* stream);
/* Tiny-M linear, R <= 16 rows: in [R, K] with row stride ld_in (0: one row for all R), w [N, K] (K % 8 == 0):
 * out = fp16(in . w + bias) (+ addend[r * ld_add + n] in fp16), replaced by fp16(SiLU(out)) with out_silu;
 * out [R, ld_out]; out2 (may be null, same layout) = fp16(SiLU(out)). */
int cfgpp_op_small_linear(const void* in, int ld_in, const void* w, const void* bias, const void* addend, int ld_add,
                          void* out, int ld_out, void* out2, int R, int N, int K, int out_silu, void* stream);
/* dst[r * ld_dst + col_off + c] = src[(r % src_rows) * cols + c], r < R, c < cols (fp16). */
int cfgpp_op_copy_rows(const void* src, int src_rows, int cols, void* dst, int ld_dst, int col_off, int R, void* stream);
/* conv_in 3x3 pad 1, 4 -> Cout (Cout % 8 == 0, W % 4 == 0): z [B,4,H,W] NCHW of z_dtype, times *in_scale_dev when
 * given (fp16 arithmetic for fp16 z), w [Cout][36] fp16, bias [Cout] -> out [reps * B, H, W, Cout] NHWC fp16, the same
 * B images written reps times. */
int cfgpp_op_conv_in(const void* z, int z_dtype, const float* in_scale_dev, const void* w, const void* bias, void* out,
                     int B, int H, int W, int Cout, int reps, void* stream);
/* conv_out 3x3 pad 1, Cin -> 4 on x [2B,H,W,Cin] NHWC fp16 (rows [0, B) uncond, [B, 2B) cond), w [4][9][Cin] fp16,
 * fused with the step `method` (CFGPP_STEP_NONE: no update; coef_host may then be null) on the state z [B,4,H,W] of
 * state_dtype. eps_uc / eps_c (may be null): the conv outputs [B,4,H,W] fp16. noise_dev / lambda_dev as in
 * cfgpp_op_cfgpp_step (lambda_dev has B entries).
 * v_ab_host (may be null: an epsilon model): (a, b) of a v-prediction model. The conv outputs (written to eps_uc / eps_c
 * as they are) are then v and become eps = fp16(fp32(a v) + fp32(b x_in)) before the step, x_in = the UNet input
 * z * (*in_scale_dev) formed as cfgpp_op_conv_in forms it (in_scale_dev may be NULL: no scaling); method must not be
 * CFGPP_STEP_NONE. Synchronises the stream. */
int cfgpp_op_conv_out_step(const void* x, const void* w, const void* bias, int B, int H, int W, int Cin, int method,
                           int state_dtype, const cfgpp_step_coef* coef_host, void* z, void* aux, void* z0t_out,
                           void* eps_uc, void* eps_c, const void* noise_dev, const float* lambda_dev,
                           const float* v_ab_host, const float* in_scale_dev, void* stream);
/* The v conversion of cfgpp_op_conv_out_step alone: eps[i] = fp16(fp32(a v[i]) + fp32(b x_in[i])), v / eps [n] fp16,
 * x_in from z [n] of z_dtype and in_scale_dev (may be NULL) as cfgpp_op_conv_in forms the UNet input. */
int cfgpp_op_v_to_eps(const void* v, const void* z, int z_dtype, const float* in_scale_dev, float a, float b, void* eps,
                      int n, void* stream);
/* nearest 2x upsample: x [B,H,W,C] NHWC fp16 (C % 8 == 0) -> out [B,2H,2W,C]. */
int cfgpp_op_upsample2x(const void* x, void* out, int B, int H, int W, int C, void* stream);
/* ControlNet conditioning image in: x [B,C,H,W] fp16 / fp32 (dtype) -> out [B,H,W,Cp] NHWC fp16, channels C..Cp-1
 * +0. */
int cfgpp_op_image_to_nhwc(const void* x, int dtype, void* out, int B, int C, int H, int W, int Cp, void* stream);
/* In-place SiLU on n fp16 values: x = fp16(x / (1 + expf(-x))) in fp32. */
int cfgpp_op_silu(void* x, size_t n, void* stream);
/* T2I-Adapter: x [B,C,H,W] fp16 / fp32 (dtype) -> out [B,H/f,W/f,C*f*f] NHWC fp16, channel c*f*f + i*f + j = fp16(x[b,
 * c, f*y+i, f*x+j]) (torch's pixel_unshuffle of fp16(x)); H, W multiples of f. */
int cfgpp_op_pixel_unshuffle(const void* x, int dtype, void* out, int B, int C, int H, int W, int f, void* stream);
/* NHWC 2x2 average pool, stride 2, even H, W: out = fp16(((x00 + x01) + x10 + x11) / 4) in fp32, C % 8 == 0. */
int cfgpp_op_avgpool2x2(const void* x, void* out, int B, int H, int W, int C, void* stream);
/* In-place ReLU on n fp16 values (x > 0 ? x : +0); out = fp16(x * s) on n fp16 values (out may be x). */
int cfgpp_op_relu(void* x, size_t n, void* stream);
int cfgpp_op_scale(const void* x, float s, void* out, size_t n, void* stream);
/* The T2I gated add: when *on_dev (int, device) is nonzero, image n of h [NB][per_image] becomes fp16(float(h) +
 * float(feat[n mod B])), feat [B][per_image]; when it is zero, nothing is written. per_image % 8 == 0. */
int cfgpp_op_t2i_add(void* h, const void* feat, int NB, int B, size_t per_image, const int* on_dev, void* stream);
/* AutoencoderKL decoder front: z [B,4,HW] of z_dtype -> fp16(w . fp16(z / scaling) + bias), w [4][4], out [B,4,HW]. */
int cfgpp_op_vae_latent_prep(const void* z, int z_dtype, float scaling, const void* w, const void* bias, void* out,
                             int B, int HW, void* stream);
/* In-place softmax of every row of s [rows, n] fp16 (n % 8 == 0) of scores * scale. */
int cfgpp_op_vae_row_softmax(void* s, int rows, int n, float scale, void* stream);
/* AutoencoderKL decoder conv_out: 3x3 pad 1, C -> 3 on x [B,H,W,C] NHWC, w [3][9][C] -> out [B,3,H,W] NCHW fp16. */
int cfgpp_op_vae_conv_rgb(const void* x, const void* w, const void* bias, void* out, int B, int H, int W, int C,
                          void* stream);
/* image [B,3,H,W] NCHW of x_dtype -> [B,4,H,W] fp16 with a zero fourth plane. */
int cfgpp_op_vae_image_pad(const void* x, int x_dtype, void* out, int B, int H, int W, void* stream);
/* AutoencoderKL encoder tail: conv_out 3x3 (C -> 8, w [8][9][C]) on x [B,H,W,C] NHWC, quant_conv (wq [8][8], bq [8]),
 * logvar clamped to [-30, 20], out [B,4,H,W] fp32 = (mean + exp(logvar / 2) * noise) * scaling; noise [B,4,H,W] fp16
 * or null (the mean). */
int cfgpp_op_vae_moments_sample(const void* x, const void* w, const void* bias, const void* wq, const void* bq,
                                const void* noise, float scaling, float* out, int B, int H, int W, int C, void* stream);
/* CLIP token + position embedding: out[r] = fp16(tok[ids[r]] + pos[r % T]), r < M; tok [vocab, D], pos [T, D]. */
int cfgpp_op_clip_embed(const int32_t* ids, const void* tok, const void* pos, void* out, int M, int T, int D, int vocab,
                        void* stream);
/* CLIP causal self-attention: qkv [B*T, 3D] (q | k | v, 64-wide heads, D = 64 heads, T <= 128) -> out [B*T, D]. */
int cfgpp_op_clip_attention(const void* qkv, void* out, int B, int T, int heads, int D, void* stream);
/* In-place CLIP MLP activation on n fp16 values (n % 8 == 0): mode 0 quick_gelu, 1 gelu (erf). */
int cfgpp_op_clip_activation(void* x, size_t n, int mode, void* stream);
/* out[b] = x[b * T + index[b]], x [B*T, D] fp16, out [B, D]. */
int cfgpp_op_clip_gather_rows(const void* x, const int32_t* index, void* out, int B, int T, int D, void* stream);
/* CLIP vision patch rows: image [B,3,S,S] fp16 / fp32 (dtype) -> out [B*(S/P)^2, Kp] fp16, row (b, py, px), column
 * (c*P + ky)*P + kx, columns 3*P*P..Kp-1 +0. */
int cfgpp_op_clip_patchify(const void* image, int dtype, void* out, int B, int S, int P, int Kp, void* stream);
/* CLIP vision embeddings: out[b, 0] = fp16(cls + pos[0]), out[b, 1 + p] = fp16(pe[b*np + p] + pos[1 + p]); pe [B*np, D],
 * cls [D], pos [np + 1, D], out [B*(np + 1), D], all fp16. */
int cfgpp_op_clip_vision_embed(const void* pe, const void* cls, const void* pos, void* out, int B, int np, int D,
                               void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CFGPP_B200_H_ */
