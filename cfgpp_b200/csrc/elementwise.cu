// cfgpp_b200 — small / HBM-bound kernels of the UNet step: timestep embeddings, tiny-M linears, conv_in, conv_out fused
// with the CFG++ guidance mix + scheduler update, nearest-2x upsample. See ops.cuh.
#include <algorithm>

#include "common.cuh"
#include "executor.cuh"
#include "ops.cuh"

namespace cfgpp {

namespace {

// ------------------------------------------------------------------------------------------------------------
// sinusoidal embedding (diffusers embeddings.get_timestep_embedding, flip_sin_to_cos=True, freq_shift=0)
// ------------------------------------------------------------------------------------------------------------
__global__ void sincos_kernel(const float* __restrict__ vals, int val_stride, int n, int dim,
                              __half* __restrict__ out, int ld, int col_off) {
  pdl_launch_dependents();
  pdl_wait();
  const int half_dim = dim >> 1;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half_dim) return;
  const int i = idx / half_dim;
  const int k = idx - i * half_dim;
  // diffusers divides the exponent by half_dim, a Python scalar, on the GPU, where torch multiplies by its fp32
  // reciprocal instead; a true division moves the frequency by up to 1 ulp of the exponent when half_dim is not a
  // power of two (320, 1280)
  const float inv_half = 1.0f / static_cast<float>(half_dim);
  const float freq = expf(__fmul_rn(-9.210340371976184f * static_cast<float>(k), inv_half));
  const float arg = vals[static_cast<size_t>(i) * val_stride] * freq;
  out[static_cast<size_t>(i) * ld + col_off + k] = __float2half_rn(cosf(arg));
  out[static_cast<size_t>(i) * ld + col_off + half_dim + k] = __float2half_rn(sinf(arg));
}

// ------------------------------------------------------------------------------------------------------------
// tiny-M linear: one warp per output feature, R <= 16 rows
// ------------------------------------------------------------------------------------------------------------
constexpr int MAX_R = 16;

__global__ void small_linear_kernel(const __half* __restrict__ in, int ld_in, const __half* __restrict__ w,
                                    const __half* __restrict__ bias, const __half* __restrict__ addend, int ld_add,
                                    __half* __restrict__ out, int ld_out, __half* __restrict__ out2, int R, int N,
                                    int K, int out_silu) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float acc[MAX_R];
#pragma unroll
  for (int r = 0; r < MAX_R; ++r) acc[r] = 0.f;
  const __half* wrow = w + static_cast<size_t>(n) * K;
  for (int k0 = lane * 8; k0 < K; k0 += 32 * 8) {
    const uint4 uw = *reinterpret_cast<const uint4*>(wrow + k0);
    const __half2* hw = reinterpret_cast<const __half2*>(&uw);
    float wf[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(hw[i]);
      wf[2 * i] = f.x;
      wf[2 * i + 1] = f.y;
    }
#pragma unroll
    for (int r = 0; r < MAX_R; ++r) {
      if (r < R) {
        const uint4 ux = *reinterpret_cast<const uint4*>(in + static_cast<size_t>(r) * ld_in + k0);
        const __half2* hx = reinterpret_cast<const __half2*>(&ux);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __half22float2(hx[i]);
          acc[r] += f.x * wf[2 * i] + f.y * wf[2 * i + 1];
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < MAX_R; ++r) {
    if (r < R) {
      float a = acc[r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) {
        if (bias) a += __half2float(bias[n]);
        __half t = __float2half_rn(a);
        if (addend) t = __float2half_rn(__half2float(t) + __half2float(addend[static_cast<size_t>(r) * ld_add + n]));
        if (out_silu) t = __float2half_rn(silu_f(__half2float(t)));
        out[static_cast<size_t>(r) * ld_out + n] = t;
        if (out2) out2[static_cast<size_t>(r) * ld_out + n] = __float2half_rn(silu_f(__half2float(t)));
      }
    }
  }
}

__global__ void copy_rows_kernel(const __half* __restrict__ src, int src_rows, int cols, __half* __restrict__ dst,
                                 int ld_dst, int col_off, int R) {
  pdl_launch_dependents();
  pdl_wait();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * cols) return;
  const int r = idx / cols, c = idx - r * cols;
  dst[static_cast<size_t>(r) * ld_dst + col_off + c] = src[static_cast<size_t>(r % src_rows) * cols + c];
}

// ------------------------------------------------------------------------------------------------------------
// conv_in: 4 -> Cout, 3x3 pad 1, NCHW latent -> NHWC fp16. thread = (pixel, 8 output channels)
// ------------------------------------------------------------------------------------------------------------
__global__ void select_step_kernel(const StepEntry* __restrict__ table, int* counter, StepArgs* args) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = *counter;
  args->cur = table[i];
  *counter = i + 1;
}

// The UNet's input value of latent element `off`: z * in_scale as conv_in forms it (fp16 arithmetic for an fp16 state,
// an fp32 product cast to fp16 for an fp32 one, as under the reference's autocast).
CFGPP_DEVICE float model_input(const void* __restrict__ z, size_t off, int z_is_half, int use_scale, float in_scale) {
  if (z_is_half) {
    __half hv = reinterpret_cast<const __half*>(z)[off];
    if (use_scale) hv = __float2half_rn(__half2float(hv) * in_scale);  // x * c_in in fp16 arithmetic
    return __half2float(hv);
  }
  float fv = reinterpret_cast<const float*>(z)[off];
  if (use_scale) fv = fv * in_scale;
  return __half2float(__float2half_rn(fv));  // autocast: conv input cast to fp16
}

// v-prediction -> epsilon for a model input x_in at the noise level abar: eps = sqrt(abar) v + sqrt(1 - abar) x_in with
// a = sqrt(abar), b = sqrt(1 - abar) — two fp32 products and an fp32 sum (no FMA contraction), rounded to fp16 as the
// model output it replaces.
CFGPP_DEVICE float v_to_eps(float v, float x_in, float a, float b) {
  return __half2float(__float2half_rn(__fadd_rn(__fmul_rn(a, v), __fmul_rn(b, x_in))));
}

__global__ void conv_in_kernel(const void* __restrict__ z, int z_is_half, const float* __restrict__ in_scale_ptr,
                               const __half* __restrict__ w, const __half* __restrict__ bias, __half* __restrict__ out,
                               int B, int H, int W, int Cout, int reps, int px_per_block,
                               const __half* __restrict__ addend) {
  pdl_launch_dependents();
  pdl_wait();
  // thread = (group of 4 horizontally adjacent pixels, 8 output channels): the 4 x 3 x 6 input patch is loaded once
  // and every weight fetched from shared memory feeds 4 pixels.
  extern __shared__ float sw[];  // [36][Cout] fp32 (tap-major: ci*9 + kh*3 + kw), then bias [Cout]
  const int use_scale = in_scale_ptr != nullptr;
  const float in_scale = use_scale ? *in_scale_ptr : 1.0f;
  for (int i = threadIdx.x; i < 36 * Cout; i += blockDim.x) {
    const int oc = i % Cout, t = i / Cout;
    sw[i] = __half2float(w[oc * 36 + t]);
  }
  for (int i = threadIdx.x; i < Cout; i += blockDim.x) sw[36 * Cout + i] = __half2float(bias[i]);
  __syncthreads();
  const int ocg_n = Cout >> 3;
  const int HW = H * W;
  const int total = B * HW;
  const int Wq = W >> 2;  // pixel quads per row (W % 4 == 0)
  for (int li = threadIdx.x; li < (px_per_block >> 2) * ocg_n; li += blockDim.x) {
    const int quad = blockIdx.x * (px_per_block >> 2) + li / ocg_n;
    const int ocg = li % ocg_n;
    if (quad * 4 >= total) break;
    const int b = quad / (H * Wq);
    const int r = quad - b * (H * Wq);
    const int h = r / Wq, x0 = (r - h * Wq) * 4;
    float acc[4][8];
#pragma unroll
    for (int px = 0; px < 4; ++px)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[px][i] = sw[36 * Cout + ocg * 8 + i];
#pragma unroll
    for (int ci = 0; ci < 4; ++ci) {
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int hh = h + kh - 1;
        float v[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) {
          const int ww = x0 + c - 1;
          float val = 0.f;
          if (hh >= 0 && hh < H && ww >= 0 && ww < W)
            val = model_input(z, (static_cast<size_t>(b) * 4 + ci) * HW + hh * W + ww, z_is_half, use_scale, in_scale);
          v[c] = val;
        }
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const float* wt = sw + (ci * 9 + kh * 3 + kw) * Cout + ocg * 8;
          float wv[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) wv[i] = wt[i];
#pragma unroll
          for (int px = 0; px < 4; ++px)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[px][i] += v[px + kw] * wv[i];
        }
      }
    }
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      uint4 o;
      o.x = pack_half2(acc[px][0], acc[px][1]);
      o.y = pack_half2(acc[px][2], acc[px][3]);
      o.z = pack_half2(acc[px][4], acc[px][5]);
      o.w = pack_half2(acc[px][6], acc[px][7]);
      const size_t pix = static_cast<size_t>(b) * HW + h * W + x0 + px;
      if (addend) {  // fp16(fp16(conv) + addend), the addend's B images shared by every repetition
        const uint4 a = *reinterpret_cast<const uint4*>(addend + pix * Cout + ocg * 8);
        const __half2* ah = reinterpret_cast<const __half2*>(&a);
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i)
          oh[i] = __floats2half2_rn(__low2float(oh[i]) + __low2float(ah[i]), __high2float(oh[i]) + __high2float(ah[i]));
      }
      for (int rep = 0; rep < reps; ++rep)
        *reinterpret_cast<uint4*>(out + (static_cast<size_t>(rep) * total + pix) * Cout + ocg * 8) = o;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// CFG++ guidance mix + scheduler update (per latent element), mirroring the reference's op-by-op rounding:
// every fp16-tensor op rounds to fp16; fp32-state ops stay un-fused fp32 (no FMA contraction).
// ------------------------------------------------------------------------------------------------------------
CFGPP_DEVICE float rh(float x) { return __half2float(__float2half_rn(x)); }  // round through fp16

template <bool kHalfState>
CFGPP_DEVICE float rs(float x) {  // round to the state dtype
  if constexpr (kHalfState) return rh(x);
  return x;
}

template <bool kHalfState>
CFGPP_DEVICE void cfgpp_update(int mode, const StepCoef& k, float lambda, float eu, float ec, float z, float old_d,
                               float noise, float& z_new, float& z0t, float& new_old) {
  // noise_pred = eps_uc + lambda * (eps_c - eps_uc)   (three fp16 tensor ops); lambda is k.lambda or the image's entry
  // of the per-image guidance table
  const float np = rh(__fadd_rn(eu, rh(__fmul_rn(lambda, rh(__fsub_rn(ec, eu))))));
  new_old = 0.f;
  if (mode == STEP_DDIM_CFGPP || mode == STEP_DDIM_INV_CFGPP || mode == STEP_DDIM_CFG) {
    // Tweedie: guided eps (CFG++ sampling, plain CFG) / eps_uc (CFG++ inversion);
    // renoise: eps_uc (CFG++ sampling) / guided eps (CFG++ inversion, plain CFG in both directions)
    const float e_tw = (mode == STEP_DDIM_INV_CFGPP) ? eu : np;
    const float e_rn = (mode == STEP_DDIM_CFGPP) ? eu : np;
    const float a = rh(__fmul_rn(k.c0, e_tw));
    z0t = rs<kHalfState>(__fdiv_rn(rs<kHalfState>(__fsub_rn(z, a)), k.c1));
    const float b = rh(__fmul_rn(k.c3, e_rn));
    z_new = rs<kHalfState>(__fadd_rn(rs<kHalfState>(__fmul_rn(k.c2, z0t)), b));
  } else {  // STEP_DPMPP2M_CFGPP (state is fp16 in the reference; kHalfState expected)
    // Family of VE-cast ("k-diffusion") updates on the Tweedie estimates  den = x - sigma eps_guided,
    // ud = x - sigma eps_uc.  k.second_order bits: 1 = second-order (2M) branch; 2 = EXTRAPOLATE with the guided
    // estimate instead of the unconditional one (plain-CFG euler / dpm++_2m: latent_diffusion.py:326-330, :470-487);
    // 4 = the 2M difference term uses the guided estimate (SD v1.5 `dpm++_2m_cfg++`, latent_diffusion.py:863, whereas
    // SDXL's `dpm++_2m_cfgpp` uses the unconditional one, latent_sdxl.py:916);
    // 8 = ancestral: add noise * sigma_up (d3) after the update (euler_a, dpm++_2s_a: latent_diffusion.py:757-760, :823);
    // 16 / 32 = the two UNet calls of a DPM-Solver++(2S) step (latent_diffusion.py:796-821): 16 parks x in `aux` and
    // leaves the midpoint x_2 as the state the next replay feeds to the UNet, 32 combines the midpoint estimates with
    // the parked x.
    const float den = rs<kHalfState>(__fadd_rn(z, rh(__fmul_rn(k.c0, np))));
    const float ud = rs<kHalfState>(__fadd_rn(z, rh(__fmul_rn(k.c0, eu))));
    const float ex = (k.second_order & 2) ? den : ud;
    z0t = den;
    new_old = ex;
    if (k.second_order & 16) {
      // x_2 = (sigma_s / sigma_t) * x - expm1(-h r) * extrap
      const float a = rs<kHalfState>(__fmul_rn(k.d0, z));
      const float b = rs<kHalfState>(__fmul_rn(k.d1, ex));
      z_new = rs<kHalfState>(__fsub_rn(a, b));
      new_old = z;
    } else if (k.second_order & 32) {
      const float xr = rs<kHalfState>(__fmul_rn(k.d1, old_d));  // (sigma_down / sigma_t) * x, x parked by the midpoint call
      if (k.second_order & 2) {
        // plain CFG: x = ratio * x - expm1(-h) * denoised_2
        z_new = rs<kHalfState>(__fsub_rn(xr, rs<kHalfState>(__fmul_rn(k.d2, den))));
      } else {
        // CFG++: x = denoised_2 - exp(-h) * uncond_denoised_2 + ratio * x
        const float t1 = rs<kHalfState>(__fmul_rn(k.d0, ud));
        z_new = rs<kHalfState>(__fadd_rn(rs<kHalfState>(__fsub_rn(den, t1)), xr));
      }
      new_old = old_d;
    } else if (!(k.second_order & 1)) {
      float d = rs<kHalfState>(__fsub_rn(z, ex));
      d = rs<kHalfState>(__fmul_rn(d, k.c1));  // / sigma_i  (scalar divisor -> reciprocal multiply on CUDA)
      d = rs<kHalfState>(__fmul_rn(d, k.c2));  // * sigma_{i+1}
      z_new = rs<kHalfState>(__fadd_rn(den, d));
    } else {
      const float df = (k.second_order & 4) ? den : ud;
      const float e1a = rs<kHalfState>(__fmul_rn(k.d0, ex));
      float e1b = rs<kHalfState>(__fmul_rn(k.d1, rs<kHalfState>(__fsub_rn(df, old_d))));
      e1b = rs<kHalfState>(__fmul_rn(e1b, k.d2));  // / (2 r)
      const float extra1 = rs<kHalfState>(__fsub_rn(e1a, e1b));
      const float extra2 = rs<kHalfState>(__fmul_rn(k.d3, z));
      z_new = rs<kHalfState>(__fadd_rn(rs<kHalfState>(__fadd_rn(den, extra1)), extra2));
    }
    if (k.second_order & 8) z_new = rs<kHalfState>(__fadd_rn(z_new, rs<kHalfState>(__fmul_rn(noise, k.d3))));
  }
}

CFGPP_DEVICE float load_state(const void* p, size_t i, bool is_half) {
  return is_half ? __half2float(reinterpret_cast<const __half*>(p)[i]) : reinterpret_cast<const float*>(p)[i];
}
CFGPP_DEVICE void store_state(void* p, size_t i, bool is_half, float v) {
  if (is_half)
    reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
  else
    reinterpret_cast<float*>(p)[i] = v;
}

CFGPP_DEVICE void apply_step_elem(int mode, int half_state, const StepArgs* args, float eu, float ec, void* z,
                                  void* aux, void* z0t_out, size_t sample_elems, size_t n, size_t i) {
  const StepCoef& k = args->cur.s.coef;
  const float* table = args->lambda;  // per-image guidance [batch]; null: the schedule's scalar
  const float lambda = table ? table[i / sample_elems] : k.lambda;
  const bool hs = half_state != 0;
  const float zv = load_state(z, i, hs);
  const bool kd = mode == STEP_DPMPP2M_CFGPP;
  const float old_d = (kd && (k.second_order & (1 | 32))) ? load_state(aux, i, hs) : 0.f;
  float noise = 0.f;
  if (kd && (k.second_order & 8)) {
    // slot index travels in c3 (exact for any realistic step count)
    const __half* base = args->noise;
    if (base) noise = __half2float(base[static_cast<size_t>(k.c3) * n + i]);
  }
  float zn, z0, no;
  if (hs)
    cfgpp_update<true>(mode, k, lambda, eu, ec, zv, old_d, noise, zn, z0, no);
  else
    cfgpp_update<false>(mode, k, lambda, eu, ec, zv, old_d, noise, zn, z0, no);
  store_state(z, i, hs, zn);
  if (z0t_out) store_state(z0t_out, i, hs, z0);
  if (mode == STEP_DPMPP2M_CFGPP && aux) store_state(aux, i, hs, no);
}

// conv_out (Cin -> 4, 3x3 pad 1) + fused step. One warp per latent pixel of image b, computing both CFG halves.
// kVPred: the conv output is v; it is converted to eps (v_to_eps with (a, b) = args->cur.v_ab and the UNet input
// rebuilt from the state z and args->cur.s.in_scale) before the step. eps_uc / eps_c receive the raw output (v) either
// way.
template <bool kVPred>
__global__ void conv_out_step_kernel(const __half* __restrict__ x, const __half* __restrict__ w,
                                     const __half* __restrict__ bias, int B, int H, int W, int Cin, int mode,
                                     int half_state, const StepArgs* __restrict__ args, void* z, void* aux,
                                     void* z0t_out, __half* __restrict__ eps_uc, __half* __restrict__ eps_c) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __half swh[];  // [4][9][Cin]
  for (int i = threadIdx.x * 8; i < 4 * 9 * Cin; i += blockDim.x * 8)
    *reinterpret_cast<uint4*>(swh + i) = *reinterpret_cast<const uint4*>(w + i);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int HW = H * W;
  const int pix = blockIdx.x * (blockDim.x >> 5) + warp;
  if (pix >= B * HW) return;
  const int b = pix / HW;
  const int r = pix - b * HW;
  const int h = r / W, xw = r - h * W;
  const int vpt = Cin >> 3;  // 8-channel vectors per tap
  float acc[2][4];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int o = 0; o < 4; ++o) acc[s][o] = 0.f;
  for (int v = lane; v < 9 * vpt; v += 32) {
    const int tap = v / vpt;
    const int c0 = (v - tap * vpt) * 8;
    const int kh = tap / 3, kw = tap - kh * 3;
    const int hh = h + kh - 1, ww = xw + kw - 1;
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
    const size_t p_uc = (static_cast<size_t>(b) * HW + hh * W + ww) * Cin + c0;
    const size_t p_c = (static_cast<size_t>(B + b) * HW + hh * W + ww) * Cin + c0;
    const uint4 u0 = *reinterpret_cast<const uint4*>(x + p_uc);
    const uint4 u1 = *reinterpret_cast<const uint4*>(x + p_c);
    const __half2* h0 = reinterpret_cast<const __half2*>(&u0);
    const __half2* h1 = reinterpret_cast<const __half2*>(&u1);
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      const uint4 uw = *reinterpret_cast<const uint4*>(swh + (o * 9 + tap) * Cin + c0);
      const __half2* hw = reinterpret_cast<const __half2*>(&uw);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 wf = __half22float2(hw[i]);
        const float2 a0 = __half22float2(h0[i]);
        const float2 a1 = __half22float2(h1[i]);
        acc[0][o] += a0.x * wf.x + a0.y * wf.y;
        acc[1][o] += a1.x * wf.x + a1.y * wf.y;
      }
    }
  }
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) acc[s][o] += __shfl_xor_sync(0xffffffffu, acc[s][o], d);
  if (lane < 4) {
    float eu = 0.f, ec = 0.f;
#pragma unroll
    for (int o = 0; o < 4; ++o)
      if (lane == o) {
        eu = acc[0][o];
        ec = acc[1][o];
      }
    const float bo = __half2float(bias[lane]);
    eu = rh(eu + bo);  // conv output is an fp16 tensor in the reference
    ec = rh(ec + bo);
    const size_t i = (static_cast<size_t>(b) * 4 + lane) * HW + r;  // NCHW latent index
    if (eps_uc) eps_uc[i] = __float2half_rn(eu);
    if (eps_c) eps_c[i] = __float2half_rn(ec);
    if constexpr (kVPred) {
      const float2 ab = args->cur.v_ab;
      const float x_in = model_input(z, i, half_state, 1, args->cur.s.in_scale);
      eu = v_to_eps(eu, x_in, ab.x, ab.y);
      ec = v_to_eps(ec, x_in, ab.x, ab.y);
    }
    if (mode != STEP_NONE)
      apply_step_elem(mode, half_state, args, eu, ec, z, aux, z0t_out, static_cast<size_t>(4) * HW,
                      static_cast<size_t>(B) * 4 * HW, i);
  }
}

__global__ void v_to_eps_kernel(const __half* __restrict__ v, const void* __restrict__ z, int z_is_half,
                                const float* __restrict__ in_scale_ptr, float a, float b, __half* __restrict__ eps,
                                int n) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x_in = model_input(z, i, z_is_half, in_scale_ptr != nullptr, in_scale_ptr ? *in_scale_ptr : 1.0f);
  eps[i] = __float2half_rn(v_to_eps(__half2float(v[i]), x_in, a, b));
}

__global__ void step_only_kernel(const __half* __restrict__ eps_uc, const __half* __restrict__ eps_c, int n, int mode,
                                 int half_state, const StepArgs* __restrict__ args, void* z, void* aux, void* z0t_out,
                                 int sample_elems) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  apply_step_elem(mode, half_state, args, __half2float(eps_uc[i]), __half2float(eps_c[i]), z, aux, z0t_out,
                  sample_elems, n, i);
}

// ------------------------------------------------------------------------------------------------------------
// resampling helpers (NHWC fp16, 16-byte vectors)
// ------------------------------------------------------------------------------------------------------------
__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int H, int W, int Cv) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t total = static_cast<size_t>(B) * 4 * H * W * Cv;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = i % Cv;
    size_t t = i / Cv;
    const int ow = t % (2 * W);
    t /= (2 * W);
    const int oh = t % (2 * H);
    const int b = t / (2 * H);
    out[i] = x[((static_cast<size_t>(b) * H + (oh >> 1)) * W + (ow >> 1)) * Cv + cv];
  }
}

}  // namespace

void run_sincos_embed(const float* vals, int val_stride, int n, int dim, __half* out, int ld, int col_off,
                      cudaStream_t stream) {
  const int total = n * (dim / 2);
  launch_pdl(sincos_kernel, dim3((total + 255) / 256), dim3(256), 0, stream, vals, val_stride, n, dim, out, ld, col_off);
}

void run_small_linear(const __half* in, int ld_in, const __half* w, const __half* bias, const __half* addend,
                      int ld_add, __half* out, int ld_out, __half* out2, int R, int N, int K, bool out_silu,
                      cudaStream_t stream) {
  CFGPP_REQUIRE(R >= 1 && R <= MAX_R, "small_linear supports 1..16 rows");
  CFGPP_REQUIRE(K % 8 == 0 && ld_in % 8 == 0, "small_linear needs K % 8 == 0");
  const int warps = 8;
  launch_pdl(small_linear_kernel, dim3((N + warps - 1) / warps), dim3(warps * 32), 0, stream, in, ld_in, w, bias, addend, ld_add, out,
                                                                          ld_out, out2, R, N, K, out_silu ? 1 : 0);
}

void run_copy_rows(const __half* src, int src_rows, int cols, __half* dst, int ld_dst, int col_off, int R,
                   cudaStream_t stream) {
  const int total = R * cols;
  launch_pdl(copy_rows_kernel, dim3((total + 255) / 256), dim3(256), 0, stream, src, src_rows, cols, dst, ld_dst, col_off, R);
}

void run_select_step(const StepEntry* table, int* counter, StepArgs* args, cudaStream_t stream) {
  launch_pdl(select_step_kernel, dim3(1), dim3(1), 0, stream, table, counter, args);
}

void run_conv_in(const void* z, int z_is_half, const float* in_scale, const __half* w, const __half* bias,
                 __half* out, int B, int H, int W, int Cout, int reps, cudaStream_t stream, const __half* addend) {
  CFGPP_REQUIRE(Cout % 8 == 0 && W % 4 == 0, "conv_in needs Cout % 8 == 0 and W % 4 == 0");
  const int ppb = 128;
  const size_t smem = (36 * Cout + Cout) * sizeof(float);
  static bool configured = false;
  if (!configured && smem > 48 * 1024) {
    CFGPP_CHECK_CUDA(cudaFuncSetAttribute(conv_in_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    configured = true;
  }
  const int total = B * H * W;
  launch_pdl(conv_in_kernel, dim3((total + ppb - 1) / ppb), dim3(320), smem, stream, z, z_is_half, in_scale, w, bias, out, B, H, W, Cout,
                                                                 reps, ppb, addend);
}

// ------------------------------------------------------------------------------------------------------------
// ControlNet conditioning embedding: the image in, with its channels zero-padded to the count the implicit-GEMM
// convolution takes (exact: padded channels are zero in and zero out), and a SiLU pass
// ------------------------------------------------------------------------------------------------------------
__global__ void image_to_nhwc_kernel(const void* __restrict__ x, int x_is_half, __half* __restrict__ out, int B, int C,
                                     int HW, int Cp) {
  const size_t n = static_cast<size_t>(B) * HW * Cp;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = i % Cp;
    const size_t pix = i / Cp;
    const size_t b = pix / HW, p = pix % HW;
    __half v = __float2half(0.f);
    if (c < C) {
      const size_t src = (b * C + c) * HW + p;
      v = x_is_half ? reinterpret_cast<const __half*>(x)[src] : __float2half_rn(reinterpret_cast<const float*>(x)[src]);
    }
    out[i] = v;
  }
}

__global__ void silu_kernel(__half* __restrict__ x, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float v = __half2float(x[i]);
    x[i] = __float2half_rn(v / (1.0f + expf(-v)));
  }
}

void run_image_to_nhwc(const void* x, int x_is_half, __half* out, int B, int C, int H, int W, int Cp,
                       cudaStream_t stream) {
  const size_t n = static_cast<size_t>(B) * H * W * Cp;
  image_to_nhwc_kernel<<<grid_for(n), 256, 0, stream>>>(x, x_is_half, out, B, C, H * W, Cp);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

void run_silu(__half* x, size_t n, cudaStream_t stream) {
  silu_kernel<<<grid_for(n), 256, 0, stream>>>(x, n);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

// The state dtype travels in bit 8 of `mode` (mode | 0x100 = fp16 sampler state).
void run_conv_out_step(const __half* x, const __half* w, const __half* bias, int B, int H, int W, int Cin, int mode,
                       const StepArgs* args, void* z, void* aux, void* z0t_out, __half* eps_uc, __half* eps_c,
                       cudaStream_t stream, bool v_pred) {
  CFGPP_REQUIRE(Cin % 8 == 0, "conv_out Cin must be a multiple of 8");
  const int half_state = (mode & 0x100) ? 1 : 0;
  const int m = mode & 0xff;
  const size_t smem = static_cast<size_t>(4) * 9 * Cin * sizeof(__half);
  CFGPP_REQUIRE(smem <= 48 * 1024, "conv_out weights must fit 48 KB of shared memory");
  const int warps = 8;
  const int total = B * H * W;
  const dim3 grid((total + warps - 1) / warps), block(warps * 32);
  if (v_pred && m != STEP_NONE)
    launch_pdl(conv_out_step_kernel<true>, grid, block, smem, stream, x, w, bias, B, H, W, Cin, m, half_state, args, z,
               aux, z0t_out, eps_uc, eps_c);
  else
    launch_pdl(conv_out_step_kernel<false>, grid, block, smem, stream, x, w, bias, B, H, W, Cin, m, half_state, args,
               z, aux, z0t_out, eps_uc, eps_c);
}

void run_v_to_eps(const __half* v, const void* z, int z_is_half, const float* in_scale, float a, float b, __half* eps,
                  int n, cudaStream_t stream) {
  launch_pdl(v_to_eps_kernel, dim3((n + 255) / 256), dim3(256), 0, stream, v, z, z_is_half, in_scale, a, b, eps, n);
}

void run_step_only(const __half* eps_uc, const __half* eps_c, int n, int mode, const StepArgs* args, void* z,
                   void* aux, void* z0t_out, int sample_elems, cudaStream_t stream) {
  CFGPP_REQUIRE(sample_elems > 0 && n % sample_elems == 0,
                "the step needs the per-image element count (a divisor of n) for a guidance table");
  const int half_state = (mode & 0x100) ? 1 : 0;
  launch_pdl(step_only_kernel, dim3((n + 255) / 256), dim3(256), 0, stream, eps_uc, eps_c, n, mode & 0xff, half_state,
             args, z, aux, z0t_out, sample_elems);
}

void run_upsample2x(const __half* x, __half* out, int B, int H, int W, int C, cudaStream_t stream) {
  CFGPP_REQUIRE(C % 8 == 0, "upsample C % 8");
  const size_t total = static_cast<size_t>(B) * 4 * H * W * (C / 8);
  const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, num_sms() * 16));
  launch_pdl(upsample2x_kernel, dim3(blocks), dim3(256), 0, stream, reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), B, H,
                                                W, C / 8);
}

}  // namespace cfgpp
