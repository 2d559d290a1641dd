// cfgpp_b200 — C ABI, operator-level entry points (one call = one kernel launch on the caller's stream).
// Declared in include/cfgpp_b200.h. No C++ exception crosses the boundary: every entry point returns an int
// status (0 = OK) and records a message retrievable with cfgpp_last_error().
#include <cstring>

#include "capi_util.h"
#include "attention.cuh"
#include "executor.cuh"
#include "gemm.cuh"
#include "ops.cuh"
#include "../../include/cfgpp_b200.h"

using namespace cfgpp;

extern "C" {

CFGPP_API int cfgpp_op_linear(const void* a, int lda, const void* a2, int lda2, int k_split, const void* w, int M,
                              int N, int K, const void* bias, const void* addend, int ld_add,
                              int add_rows_per_group, void* out, int ldc, int geglu, int force_bn, int force_streamk,
                              void* stream) {
  return guarded([&] {
    GemmOp op = make_linear_op((const __half*)a, lda, (const __half*)a2, lda2, k_split, (const __half*)w, M, N, K,
                               (const __half*)bias, (const __half*)addend, ld_add, add_rows_per_group, (__half*)out,
                               ldc, geglu != 0, force_bn, force_streamk != 0);
    run_gemm_op(op, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_linear_lnfold(const void* a, const void* w, int M, int N, int K, const void* bias,
                                     const void* addend, int ld_add, int add_rows_per_group, void* out, int ldc,
                                     int geglu, int force_bn, int force_streamk, float* stats_out, const float* stats_in,
                                     int ln_parts, float ln_eps, const float* ln_s, const float* ln_t, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE((stats_out != nullptr) != (stats_in != nullptr), "exactly one of stats_out / stats_in");
    CFGPP_REQUIRE(stats_out == nullptr || force_bn != 0, "a statistics producer needs an explicit tile width");
    CFGPP_REQUIRE(stats_in == nullptr || (ln_parts >= 1 && ln_s && ln_t), "a LayerNorm-fold consumer needs parts, s, t");
    GemmOp op = make_linear_op((const __half*)a, K, nullptr, 0, 0, (const __half*)w, M, N, K, (const __half*)bias,
                               (const __half*)addend, ld_add, add_rows_per_group, (__half*)out, ldc, geglu != 0,
                               force_bn, force_streamk != 0);
    op.p.stats_out = stats_out;
    if (stats_in) {
      op.p.stats_in = stats_in;
      op.p.ln_parts = ln_parts;
      op.p.ln_inv_c = 1.0f / static_cast<float>(K);
      op.p.ln_eps = ln_eps;
      op.p.ln_s = ln_s;
      op.p.ln_t = ln_t;
    }
    run_gemm_op(op, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_linear_scaled_residual(const void* a, const void* w, int M, int N, int K, const void* bias,
                                              const void* addend, const float* scale_dev, void* out, int force_bn,
                                              void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(addend != nullptr, "the scaled residual epilogue needs an addend");
    GemmOp op = make_linear_op((const __half*)a, K, nullptr, 0, 0, (const __half*)w, M, N, K, (const __half*)bias,
                               (const __half*)addend, N, 1, (__half*)out, N, false, force_bn);
    op.p.res_scale = scale_dev;
    run_gemm_op(op, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_fold_ln(const void* w, const void* gamma, const void* beta, const void* bias, void* wf,
                               float* s, float* t, int N, int K, void* stream) {
  return guarded([&] {
    run_fold_ln((const __half*)w, (const __half*)gamma, (const __half*)beta, (const __half*)bias, (__half*)wf, s, t, N,
                K, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_lora_merge(const void* base, const void* const* downs, const void* const* ups, const int* ranks,
                                  const float* coefs_host, int n_adapters, int N, int K, void* out, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(n_adapters >= 0 && n_adapters <= kMaxLoraPerTarget, "at most 4 adapters merge into one weight");
    LoraMergeArgs a{};
    a.n = n_adapters;
    for (int i = 0; i < n_adapters; ++i) {
      a.down[i] = (const __half*)downs[i];
      a.up[i] = (const __half*)ups[i];
      a.rank[i] = ranks[i];
      a.coef[i] = coefs_host[i];
    }
    run_lora_merge((const __half*)base, a, N, K, (__half*)out, (cudaStream_t)stream);
  });
}

// Debug aid (not in the public header): run the linear op `iters` times and return per-CTA timestamps of the last run.
CFGPP_API int cfgpp_dbg_linear_timeline(const void* a, int lda, const void* w, int M, int N, int K, const void* bias,
                                        const void* addend, void* out, int force_bn, int iters,
                                        unsigned long long* host_out /*[grid][16]*/, int* grid_out, void* stream) {
  return guarded([&] {
    GemmOp op = make_linear_op((const __half*)a, lda, nullptr, 0, 0, (const __half*)w, M, N, K, (const __half*)bias,
                               (const __half*)addend, N, 1, (__half*)out, N, false, force_bn);
    unsigned long long* d = nullptr;
    CFGPP_CHECK_CUDA(cudaMalloc(&d, sizeof(unsigned long long) * 16 * op.grid));
    CFGPP_CHECK_CUDA(cudaMemset(d, 0, sizeof(unsigned long long) * 16 * op.grid));
    op.p.timeline = d;
    for (int i = 0; i < iters; ++i) run_gemm_op(op, (cudaStream_t)stream);
    CFGPP_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    CFGPP_CHECK_CUDA(cudaMemcpy(host_out, d, sizeof(unsigned long long) * 16 * op.grid, cudaMemcpyDeviceToHost));
    *grid_out = op.grid;
    cudaFree(d);
  });
}

// Debug aid (not in the public header): the schedule cfgpp_op_linear (conv == 0) or cfgpp_op_conv3x3_ex (conv == 1)
// would run with these arguments, without launching it. The conv arguments are ignored for a linear op and the
// linear-only ones (a2, lda2, k_split, K, ldc, geglu, force_streamk) for a convolution; M, N are the conv's B, Cout and
// lda its Cin. info[8] = {bn, grid, tiles, streamk, sk_tiles, max_pieces, a_mode, k_blocks} (GemmSchedule).
CFGPP_API int cfgpp_dbg_gemm_schedule(int conv, const void* a, int lda, const void* a2, int lda2, int k_split,
                                      const void* w, int M, int N, int K, const void* bias, const void* addend,
                                      int ld_add, int add_rows_per_group, void* out, int ldc, int geglu, int force_bn,
                                      int force_streamk, int H, int W, int stride, int pad, int force_im2col,
                                      int* info) {
  return guarded([&] {
    GemmOp op = conv ? make_conv3x3_op((const __half*)a, M, H, W, lda, (const __half*)w, N, (const __half*)bias,
                                       (const __half*)addend, ld_add, add_rows_per_group, (__half*)out, force_bn,
                                       stride, pad, force_im2col != 0)
                     : make_linear_op((const __half*)a, lda, (const __half*)a2, lda2, k_split, (const __half*)w, M, N,
                                      K, (const __half*)bias, (const __half*)addend, ld_add, add_rows_per_group,
                                      (__half*)out, ldc, geglu != 0, force_bn, force_streamk != 0);
    const GemmSchedule s = gemm_schedule(op);
    const int v[8] = {s.bn, s.grid, s.tiles, s.streamk, s.sk_tiles, s.max_pieces, s.a_mode, s.k_blocks};
    for (int i = 0; i < 8; ++i) info[i] = v[i];
  });
}

CFGPP_API int cfgpp_op_conv3x3(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias,
                               const void* addend, int ld_add, int add_rows_per_group, void* out, int force_bn,
                               void* stream) {
  return guarded([&] {
    GemmOp op = make_conv3x3_op((const __half*)x, B, H, W, Cin, (const __half*)w, Cout, (const __half*)bias,
                                (const __half*)addend, ld_add, add_rows_per_group, (__half*)out, force_bn);
    run_gemm_op(op, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_conv3x3_s2(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias,
                                  int pad, void* out, void* stream) {
  return guarded([&] {
    GemmOp op = make_conv3x3_op((const __half*)x, B, H, W, Cin, (const __half*)w, Cout, (const __half*)bias, nullptr, 0, 1,
                                (__half*)out, 0, 2, pad);
    run_gemm_op(op, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_conv3x3_ex(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias,
                                  const void* addend, int ld_add, int add_rows_per_group, void* out, int force_bn,
                                  int stride, int pad, int force_im2col, void* stream) {
  return guarded([&] {
    GemmOp op = make_conv3x3_op((const __half*)x, B, H, W, Cin, (const __half*)w, Cout, (const __half*)bias,
                                (const __half*)addend, ld_add, add_rows_per_group, (__half*)out, force_bn, stride, pad,
                                force_im2col != 0);
    run_gemm_op(op, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_attention(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out,
                                 int ldo, int B, int H, int Nq, int Nkv, int head_dim, void* stream) {
  return guarded([&] {
    AttnOp op = make_attn_op((const __half*)q, ldq, (const __half*)k, ldk, (const __half*)v, ldv, (__half*)out, ldo,
                             B, H, Nq, Nkv, head_dim);
    run_attn_op(op, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_attention_ip(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv,
                                    const void* k2, int ldk2, const void* v2, int ldv2, int Nkv2,
                                    const float* ip_scale_dev, void* out, int ldo, int B, int H, int Nq, int Nkv,
                                    int head_dim, void* stream) {
  return guarded([&] {
    AttnOp op = make_attn_ip_op((const __half*)q, ldq, (const __half*)k, ldk, (const __half*)v, ldv, (const __half*)k2,
                                ldk2, (const __half*)v2, ldv2, Nkv2, ip_scale_dev, (__half*)out, ldo, B, H, Nq, Nkv,
                                head_dim);
    run_attn_op(op, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_groupnorm(const void* x1, int C1, const void* x2, int C2, int B, int HW, const void* gamma,
                                 const void* beta, float eps, int silu, void* out, void* stream) {
  return guarded([&] {
    float* partial = nullptr;
    CFGPP_CHECK_CUDA(cudaMalloc(&partial, gn_partial_floats(B, HW) * sizeof(float)));
    try {
      run_groupnorm((const __half*)x1, C1, (const __half*)x2, C2, B, HW, (const __half*)gamma, (const __half*)beta,
                    eps, silu != 0, partial, (__half*)out, (cudaStream_t)stream);
    } catch (...) {
      cudaFree(partial);
      throw;
    }
    CFGPP_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));  // test-only entry point: scratch freed below
    cudaFree(partial);
  });
}

CFGPP_API int cfgpp_op_layernorm(const void* x, int M, int C, const void* gamma, const void* beta, float eps,
                                 void* out, void* stream) {
  return guarded([&] {
    run_layernorm((const __half*)x, M, C, (const __half*)gamma, (const __half*)beta, eps, (__half*)out,
                  (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_ip_ln_concat(const void* x, const void* lat, int NB, int T, int Q, int C, const void* g0,
                                    const void* b0, const void* g1, const void* b1, float eps, void* kv, void* q,
                                    void* stream) {
  return guarded([&] {
    run_ln_concat((const __half*)x, (const __half*)lat, NB, T, Q, C, (const __half*)g0, (const __half*)b0,
                  (const __half*)g1, (const __half*)b1, eps, (__half*)kv, (__half*)q, (cudaStream_t)stream);
  });
}

}  // extern "C"

namespace {
// Runs one step launch `launch(args_dev)` on a scratch device copy of `args`, then synchronises and frees it.
// in_scale_dev (may be null: 1.0, which leaves the model input exact): the entry's input scale, copied on the device.
template <class Launch>
void with_step_block(const StepArgs& args, const float* in_scale_dev, cudaStream_t stream, Launch&& launch) {
  StepArgs* dev = nullptr;
  CFGPP_CHECK_CUDA(cudaMalloc(&dev, sizeof(StepArgs)));
  cudaError_t e = cudaMemcpyAsync(dev, &args, sizeof(StepArgs), cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess && in_scale_dev)
    e = cudaMemcpyAsync(&dev->cur.s.in_scale, in_scale_dev, sizeof(float), cudaMemcpyDeviceToDevice, stream);
  if (e == cudaSuccess) {
    try {
      launch(const_cast<const StepArgs*>(dev));
    } catch (...) {
      cudaFree(dev);
      throw;
    }
    e = cudaStreamSynchronize(stream);  // test-only entry point: scratch freed below
  }
  cudaFree(dev);
  CFGPP_CHECK_CUDA(e);
}

// The record of one op-level step: coefficients (zeros when coef_host is null), in_scale 1, the two tables.
StepArgs step_args(const cfgpp_step_coef* coef_host, const void* noise_dev, const float* lambda_dev) {
  static_assert(sizeof(cfgpp_step_coef) == sizeof(StepCoef), "ABI struct mismatch");
  StepArgs a{};
  if (coef_host) std::memcpy(&a.cur.s.coef, coef_host, sizeof(StepCoef));
  a.cur.s.in_scale = 1.0f;
  a.noise = static_cast<const __half*>(noise_dev);
  a.lambda = lambda_dev;
  return a;
}
}  // namespace

extern "C" {

CFGPP_API int cfgpp_op_cfgpp_step(const void* eps_uc, const void* eps_c, int n, int method, int state_dtype,
                                  const cfgpp_step_coef* coef_host, void* z, void* aux, void* z0t_out,
                                  const void* noise_dev, const float* lambda_dev, int batch, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(!lambda_dev || (batch >= 1 && n % batch == 0), "guidance table: batch must divide n");
    CFGPP_REQUIRE(coef_host != nullptr, "the step needs its coefficients");
    const cudaStream_t st = (cudaStream_t)stream;
    with_step_block(step_args(coef_host, noise_dev, lambda_dev), nullptr, st, [&](const StepArgs* args) {
      run_step_only((const __half*)eps_uc, (const __half*)eps_c, n, method | (state_dtype == CFGPP_F16 ? 0x100 : 0),
                    args, z, aux, z0t_out, lambda_dev ? n / batch : n, st);
    });
  });
}

CFGPP_API int cfgpp_op_timestep_embedding(const float* vals, int val_stride, int n, int dim, void* out, int ld,
                                          int col_off, void* stream) {
  return guarded([&] {
    run_sincos_embed(vals, val_stride, n, dim, (__half*)out, ld, col_off, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_small_linear(const void* in, int ld_in, const void* w, const void* bias, const void* addend,
                                    int ld_add, void* out, int ld_out, void* out2, int R, int N, int K, int out_silu,
                                    void* stream) {
  return guarded([&] {
    run_small_linear((const __half*)in, ld_in, (const __half*)w, (const __half*)bias, (const __half*)addend, ld_add,
                     (__half*)out, ld_out, (__half*)out2, R, N, K, out_silu != 0, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_copy_rows(const void* src, int src_rows, int cols, void* dst, int ld_dst, int col_off, int R,
                                 void* stream) {
  return guarded([&] {
    run_copy_rows((const __half*)src, src_rows, cols, (__half*)dst, ld_dst, col_off, R, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_conv_in(const void* z, int z_dtype, const float* in_scale_dev, const void* w, const void* bias,
                               void* out, int B, int H, int W, int Cout, int reps, void* stream) {
  return guarded([&] {
    run_conv_in(z, z_dtype == CFGPP_F16 ? 1 : 0, in_scale_dev, (const __half*)w, (const __half*)bias, (__half*)out, B,
                H, W, Cout, reps, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_conv_in_add(const void* z, int z_dtype, const float* in_scale_dev, const void* w,
                                   const void* bias, const void* addend, void* out, int B, int H, int W, int Cout,
                                   int reps, void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(addend != nullptr, "null addend");
    run_conv_in(z, z_dtype == CFGPP_F16 ? 1 : 0, in_scale_dev, (const __half*)w, (const __half*)bias, (__half*)out, B,
                H, W, Cout, reps, (cudaStream_t)stream, (const __half*)addend);
  });
}

CFGPP_API int cfgpp_op_conv_out_step(const void* x, const void* w, const void* bias, int B, int H, int W, int Cin,
                                     int method, int state_dtype, const cfgpp_step_coef* coef_host, void* z, void* aux,
                                     void* z0t_out, void* eps_uc, void* eps_c, const void* noise_dev,
                                     const float* lambda_dev, const float* v_ab_host, const float* in_scale_dev,
                                     void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(method == CFGPP_STEP_NONE || coef_host != nullptr, "a step method needs its coefficients");
    CFGPP_REQUIRE(!v_ab_host || (method != CFGPP_STEP_NONE && z != nullptr),
                  "the v conversion belongs to a step: method, coefficients and state");
    StepArgs a = step_args(coef_host, noise_dev, lambda_dev);
    if (v_ab_host) a.cur.v_ab = make_float2(v_ab_host[0], v_ab_host[1]);
    const cudaStream_t st = (cudaStream_t)stream;
    with_step_block(a, in_scale_dev, st, [&](const StepArgs* args) {
      run_conv_out_step((const __half*)x, (const __half*)w, (const __half*)bias, B, H, W, Cin,
                        method | (state_dtype == CFGPP_F16 ? 0x100 : 0), args, z, aux, z0t_out, (__half*)eps_uc,
                        (__half*)eps_c, st, v_ab_host != nullptr);
    });
  });
}

CFGPP_API int cfgpp_op_v_to_eps(const void* v, const void* z, int z_dtype, const float* in_scale_dev, float a, float b,
                                void* eps, int n, void* stream) {
  return guarded([&] {
    run_v_to_eps((const __half*)v, z, z_dtype == CFGPP_F16 ? 1 : 0, in_scale_dev, a, b, (__half*)eps, n,
                 (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_upsample2x(const void* x, void* out, int B, int H, int W, int C, void* stream) {
  return guarded([&] { run_upsample2x((const __half*)x, (__half*)out, B, H, W, C, (cudaStream_t)stream); });
}

CFGPP_API int cfgpp_op_image_to_nhwc(const void* x, int dtype, void* out, int B, int C, int H, int W, int Cp,
                                     void* stream) {
  return guarded([&] {
    CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "image: fp16 or fp32");
    CFGPP_REQUIRE(C >= 1 && Cp >= C, "the padded channel count must hold the image's channels");
    run_image_to_nhwc(x, dtype == CFGPP_F16, (__half*)out, B, C, H, W, Cp, (cudaStream_t)stream);
  });
}

CFGPP_API int cfgpp_op_silu(void* x, size_t n, void* stream) {
  return guarded([&] { run_silu((__half*)x, n, (cudaStream_t)stream); });
}

}  // extern "C"
