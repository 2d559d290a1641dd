// cfgpp_b200 — host entry points of the non-GEMM kernels (norms, embeddings, conv_in / conv_out + fused CFG++ step,
// resampling helpers). All enqueue on the given stream, never synchronise, and are CUDA-graph capturable.
#pragma once
#include "host.h"

namespace cfgpp {

// ---- norm.cu -----------------------------------------------------------------------------------------------
int gn_px_per_block(int HW);
int gn_num_chunks(int HW);
size_t gn_partial_floats(int B, int HW);
// GroupNorm(32) over channel-concat [x1 | x2] (x2 may be null), NHWC, optional SiLU. out [B,HW,C1+C2] fp16.
void run_groupnorm(const __half* x1, int C1, const __half* x2, int C2, int B, int HW, const __half* gamma,
                   const __half* beta, float eps, bool silu, float* partial, __half* out, cudaStream_t stream);
void run_layernorm(const __half* x, int M, int C, const __half* gamma, const __half* beta, float eps, __half* out,
                   cudaStream_t stream);
// The two LayerNorms of one IP-Adapter Plus Resampler layer: kv [NB][T + Q][C] holds LN0(x[b]) (x [NB][T][C]) in its
// first T rows per image and LN1(lat[b]) (lat [NB][Q][C]) in the last Q, and q [NB][Q][C] gets LN1(lat) again. Every
// row is bit-identical to run_layernorm's output for it.
void run_ln_concat(const __half* x, const __half* lat, int NB, int T, int Q, int C, const __half* g0, const __half* b0,
                   const __half* g1, const __half* b1, float eps, __half* kv, __half* q, cudaStream_t stream);
// LayerNorm fold of a weight w [N][K] (see GemmParams): wf = fp16(w * gamma), s[n] = sum_k wf[n,k],
// t[n] = sum_k beta[k] w[n,k] + bias[n] (bias may be null); s, t fp32.
void run_fold_ln(const __half* w, const __half* gamma, const __half* beta, const __half* bias, __half* wf, float* s,
                 float* t, int N, int K, cudaStream_t stream);

// ---- elementwise.cu ----------------------------------------------------------------------------------------
// diffusers get_timestep_embedding(flip_sin_to_cos=True, shift 0): out[i, col_off + (cos | sin)], fp16.
// value i is read at vals[i * val_stride] and written to row i.
void run_sincos_embed(const float* vals, int val_stride, int n, int dim, __half* out, int ld, int col_off,
                      cudaStream_t stream);
// out[r, n] = fp16(acc + bias[n]) (+ addend[r, n] in fp16 arithmetic); optional out_silu (replace by SiLU) and
// out2 = SiLU(out) copy. R <= 16 rows; weight [N][K] fp16, K % 8 == 0.
void run_small_linear(const __half* in, int ld_in, const __half* w, const __half* bias, const __half* addend,
                      int ld_add, __half* out, int ld_out, __half* out2, int R, int N, int K, bool out_silu,
                      cudaStream_t stream);
// copy rows: dst[r, col_off + c] = src[r % src_rows, c]  (fp16) — used to assemble the add-embedding input
void run_copy_rows(const __half* src, int src_rows, int cols, __half* dst, int ld_dst, int col_off, int R,
                   cudaStream_t stream);

// conv_in 3x3 pad 1, Cin = 4: z [B,4,H,W] (fp32 or fp16 NCHW, optionally scaled by in_scale in fp16 arithmetic)
// -> NHWC fp16 [reps*B, H, W, Cout]; the same result is written `reps` times (uncond and cond halves share z).
// in_scale (device pointer, may be null): model input is z * (*in_scale) — the DPM++ `x * c_in` (latent_sdxl.py:901).
// addend (may be null): [B, H, W, Cout] NHWC fp16, added to every repetition as fp16(fp16(conv) + addend) — the
// ControlNet's `sample + cond`.
void run_conv_in(const void* z, int z_is_half, const float* in_scale, const __half* w /*[Cout][36]*/,
                 const __half* bias, __half* out, int B, int H, int W, int Cout, int reps, cudaStream_t stream,
                 const __half* addend = nullptr);
// ControlNet conditioning embedding helpers: image [B,C,H,W] NCHW (fp16 or fp32) -> fp16 NHWC [B,H,W,Cp] with zero
// channels C..Cp-1; in-place fp16(SiLU(x)) over n values. Its convolutions' weights and biases are zero-padded to
// [Cout_p][9][Cin_p] and [Cout_p] by the weight store (WeightStore::packed_conv3x3 and packed_heads_rows).
void run_image_to_nhwc(const void* x, int x_is_half, __half* out, int B, int C, int H, int W, int Cp,
                       cudaStream_t stream);
void run_silu(__half* x, size_t n, cudaStream_t stream);

// ---- t2i_adapter.cu ----------------------------------------------------------------------------------------
// image [B,C,H,W] NCHW (fp16 or fp32) -> NHWC fp16 [B,H/f,W/f,C*f*f], channel c*f*f + i*f + j = x[b,c,f*y+i,f*x+j]
void run_pixel_unshuffle(const void* x, int x_is_half, __half* out, int B, int C, int H, int W, int f,
                         cudaStream_t stream);
// NHWC 2x2 / stride-2 average pool over even H, W: fp16(((x00 + x01) + x10 + x11) / 4) in fp32 (torch's order)
void run_avgpool2x2(const __half* x, __half* out, int B, int H, int W, int C, cudaStream_t stream);
void run_relu(__half* x, size_t n, cudaStream_t stream);                        // in place, x > 0 ? x : +0
void run_scale(const __half* x, float s, __half* out, size_t n, cudaStream_t stream);  // fp16(float(x) * s)
// The T2I-Adapter's add into the UNet's down path, a launch of the step graph: when *on != 0, image n of h
// [NB][per_image] becomes fp16(float(h) + float(feat[n % B])); when *on == 0 nothing is written. per_image % 8 == 0.
void run_t2i_add(__half* h, const __half* feat, int NB, int B, size_t per_image, const int* on, cudaStream_t stream);

enum StepMode : int {
  STEP_NONE = 0,        // only emit eps_uc / eps_c (the predict_noise seam)
  STEP_DDIM_CFGPP = 1,  // latent_diffusion.py:660-666, latent_sdxl.py:738-744 (fp32 state)
  STEP_DDIM_INV_CFGPP = 2,  // latent_diffusion.py:904-908 (fp32 state)
  STEP_DPMPP2M_CFGPP = 3,   // latent_sdxl.py:902-919 (fp16 state, keeps old_denoised)
  STEP_DDIM_CFG = 4,        // plain-CFG DDIM step / inversion step: Tweedie AND renoise with the guided eps
                            // (latent_diffusion.py:283-287, :176-177; latent_sdxl.py:451-455, :321-322)
};

struct StepCoef {  // per-step scalars, computed on the host in fp32 exactly as the reference does
  float lambda;    // cfg_guidance
  float c0, c1, c2, c3;  // DDIM: sqrt(1-at), sqrt(at), sqrt(at_next), sqrt(1-at_next)
                         // DDIM-inv: sqrt(1-at_prev), sqrt(at_prev), sqrt(at), sqrt(1-at)
                         // DPM++: c_out(-sigma_i), 1/sigma_i, sigma_{i+1}, unused
  float d0, d1, d2;      // DPM++ 2M branch: -exp(-h), expm1(-h), 1/(2r) ; d3 = exp(-h)
  float d3;
  int second_order;      // DPM++ / Euler family bits: 1 = 2M update (else Euler), 2 = extrapolate with the guided
                         // estimate (plain CFG), 4 = 2M difference term on the guided estimate (SD v1.5 dpm++_2m_cfg++),
                         // 8 = ancestral noise: + noise[slot c3] * d3 (sigma_up), 16 / 32 = midpoint / final call of a
                         // DPM-Solver++(2S) step (16: d0 = sigma_s / sigma_t, d1 = expm1(-h r); 32: d0 = exp(-h),
                         // d1 = sigma_down / sigma_t, d2 = expm1(-h))
};

// One sampler step's scalars, the layout of cfgpp_step_state.
struct StepState {
  float t;         // timestep fed to the UNet
  float in_scale;  // c_in (1.0 for DDIM)
  StepCoef coef;
};
// One schedule entry: everything a step reads that changes from step to step. A table of these lives in HBM and a
// 1-thread kernel copies the current entry into the StepArgs record, so a single CUDA graph replays for every step
// without host involvement.
struct StepEntry {
  StepState s;
  float2 v_ab;          // v-prediction (a, b) = (sqrt(abar), sqrt(1 - abar)); unused by epsilon models
  float control_scale;  // ControlNet conditioning scale
  int t2i_on;           // T2I-Adapter features added this step (nonzero) or not; fills the record's tail padding
};
static_assert(sizeof(StepEntry) == 64, "StepEntry is one 64-byte record");
// The one device record every step consumer reads (timestep embedding, conv_in, zero convs, the step kernels).
// noise: base of the ancestral noise table [slots][B,4,H,W] fp16, or null. lambda: the per-image guidance table [B]
// fp32, or null for the entry's scalar cur.s.coef.lambda. Both are read from the record, so a captured graph survives
// re-allocating, setting and clearing the tables. ip_scale: the IP-Adapter scale s every decoupled cross-attention
// launch reads (cfgpp_set_ip_adapter_scale writes it; the captured graph follows).
struct StepArgs {
  StepEntry cur;
  const __half* noise;
  const float* lambda;
  float ip_scale;
};
// args->cur = table[*counter]; ++*counter
void run_select_step(const StepEntry* table, int* counter, StepArgs* args, cudaStream_t stream);

// conv_out 3x3 (Cin -> 4) on the GroupNorm+SiLU'ed NHWC input x [2B,H,W,Cin] fused with the CFG++ guidance mix and
// the scheduler update of args->cur (args may be null for STEP_NONE). z is the sampler state (NCHW, fp32 for DDIM
// modes, fp16 for DPM++), updated in place; image b of a guidance table mixes with args->lambda[b].
// v_pred (ignored for STEP_NONE): the model predicts v. Before the step, each conv output becomes
// eps = fp16(a * v + b * x_in) with (a, b) = args->cur.v_ab and x_in the UNet input rebuilt from z and
// args->cur.s.in_scale as conv_in forms it. eps_uc / eps_c still receive the raw output v. Without v_pred the kernel is
// the epsilon-model instantiation, without any of this arithmetic.
void run_conv_out_step(const __half* x, const __half* w /*[4][9][Cin]*/, const __half* bias, int B, int H, int W,
                       int Cin, int mode, const StepArgs* args, void* z, void* aux /*old_denoised*/, void* z0t_out,
                       __half* eps_uc, __half* eps_c, cudaStream_t stream, bool v_pred = false);
// eps[i] = fp16(a * v[i] + b * x_in[i]) (the conversion of run_conv_out_step) with x_in from z [n] of z's dtype and
// *in_scale (may be null) as conv_in forms the UNet input.
void run_v_to_eps(const __half* v, const void* z, int z_is_half, const float* in_scale, float a, float b, __half* eps,
                  int n, cudaStream_t stream);

// standalone fused CFG++ update of args->cur from given eps (used when a per-step callback needs the un-fused seam);
// element i belongs to image i / sample_elems (sample_elems = 4*H*W) for args->lambda
void run_step_only(const __half* eps_uc, const __half* eps_c, int n, int mode, const StepArgs* args, void* z,
                   void* aux, void* z0t_out, int sample_elems, cudaStream_t stream);

void run_upsample2x(const __half* x, __half* out, int B, int H, int W, int C, cudaStream_t stream);

}  // namespace cfgpp
