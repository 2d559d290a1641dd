// cfgpp_b200 — the three small kernels the AutoencoderKL decoder needs beside the UNet's GEMM / conv / norm kernels
// (see vae.cuh): latent preparation (1 / scaling_factor + post_quant_conv 1x1), the row softmax of the single-head
// mid-block attention (head dim = C = 512 exceeds the flash kernel's head dims: S = Q K^T and O = P V run as
// two wgmma GEMMs around it), and conv_out (C -> 3 channels, NHWC -> NCHW).
#include "common.cuh"
#include "vae.cuh"

namespace cfgpp {

namespace {

CFGPP_DEVICE float rh(float x) { return __half2float(__float2half_rn(x)); }  // round through fp16

// z (B,4,H,W) fp32 / fp16 -> fp16( Wpq . fp16(z / s) + b )  (B,4,H,W) fp16.
// Reference: `self.vae.decode(zt / scaling_factor)` under autocast (latent_sdxl.py:163): the division happens in zt's
// dtype, post_quant_conv (fp16 weights) casts its input to fp16 and rounds its output to fp16.
__global__ void vae_latent_prep_kernel(const void* __restrict__ z, int z_is_half, float inv_is_div /*scaling*/,
                                       const __half* __restrict__ w /*[4][4]*/, const __half* __restrict__ bias,
                                       __half* __restrict__ out, int B, int HW) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  const int b = i / HW, p = i - b * HW;
  float x[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const size_t off = (static_cast<size_t>(b) * 4 + c) * HW + p;
    if (z_is_half) {
      x[c] = __half2float(__float2half_rn(__half2float(reinterpret_cast<const __half*>(z)[off]) / inv_is_div));
    } else {
      x[c] = __half2float(__float2half_rn(reinterpret_cast<const float*>(z)[off] / inv_is_div));
    }
  }
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) acc += __half2float(w[o * 4 + c]) * x[c];
    out[(static_cast<size_t>(b) * 4 + o) * HW + p] = __float2half_rn(acc + __half2float(bias[o]));
  }
}

// In-place softmax over the rows of S [rows][n] fp16: p = exp2((s - max) * scale_log2e) / sum, fp32 inside, one
// rounding to fp16 (the math path of F.scaled_dot_product_attention). One block per row; the row is re-read from
// L1 / L2 for each of the three passes (32 KB at n = 16384).
__global__ void __launch_bounds__(256) vae_row_softmax_kernel(__half* __restrict__ s, int n, float scale_log2e) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8];
  __half* row = s + static_cast<size_t>(blockIdx.x) * n;
  const int nv = n >> 3;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto block_reduce = [&](float v, bool is_max) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, v, o);
      v = is_max ? fmaxf(v, t) : v + t;
    }
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float r = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];
    return r;
  };
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(row)[v];
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      mx = fmaxf(mx, fmaxf(f.x, f.y));
    }
  }
  mx = block_reduce(mx, true);
  const float mc = mx * scale_log2e;
  float sum = 0.f;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(row)[v];
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      sum += fast_exp2(f.x * scale_log2e - mc) + fast_exp2(f.y * scale_log2e - mc);
    }
  }
  sum = block_reduce(sum, false);
  const float inv = 1.0f / sum;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(row)[v];
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      o[i] = pack_half2(fast_exp2(f.x * scale_log2e - mc) * inv, fast_exp2(f.y * scale_log2e - mc) * inv);
    }
    reinterpret_cast<uint4*>(row)[v] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// conv_out: 3x3 pad 1, C -> 3 channels on the GroupNorm+SiLU'ed NHWC input, written NCHW fp16 (B,3,H,W).
// One thread per output pixel, weights [3][9][C] in shared memory; out = fp16(acc + bias) like the reference's conv.
__global__ void __launch_bounds__(128) vae_conv_rgb_kernel(const __half* __restrict__ x, const __half* __restrict__ w,
                                                           const __half* __restrict__ bias, __half* __restrict__ out,
                                                           int B, int H, int W, int C) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __half sw[];  // [3][9][C]
  for (int i = threadIdx.x; i < 27 * C; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const size_t pix = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t HW = static_cast<size_t>(H) * W;
  if (pix >= static_cast<size_t>(B) * HW) return;
  const int b = static_cast<int>(pix / HW);
  const int r = static_cast<int>(pix - static_cast<size_t>(b) * HW);
  const int h = r / W, xw = r - h * W;
  float acc[3] = {0.f, 0.f, 0.f};
  const int cv = C >> 3;
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const int hh = h + tap / 3 - 1, ww = xw + tap % 3 - 1;
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
    const uint4* src = reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(b) * H + hh) * W + ww) * C);
    const uint4* w0 = reinterpret_cast<const uint4*>(sw + (0 * 9 + tap) * C);
    const uint4* w1 = reinterpret_cast<const uint4*>(sw + (1 * 9 + tap) * C);
    const uint4* w2 = reinterpret_cast<const uint4*>(sw + (2 * 9 + tap) * C);
    for (int v = 0; v < cv; ++v) {
      const uint4 ux = src[v], a = w0[v], bq = w1[v], cq = w2[v];
      const __half2* hx = reinterpret_cast<const __half2*>(&ux);
      const __half2* ha = reinterpret_cast<const __half2*>(&a);
      const __half2* hb = reinterpret_cast<const __half2*>(&bq);
      const __half2* hc = reinterpret_cast<const __half2*>(&cq);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 fx = __half22float2(hx[i]);
        const float2 fa = __half22float2(ha[i]), fb = __half22float2(hb[i]), fc = __half22float2(hc[i]);
        acc[0] += fx.x * fa.x + fx.y * fa.y;
        acc[1] += fx.x * fb.x + fx.y * fb.y;
        acc[2] += fx.x * fc.x + fx.y * fc.y;
      }
    }
  }
#pragma unroll
  for (int o = 0; o < 3; ++o)
    out[(static_cast<size_t>(b) * 3 + o) * HW + r] = __float2half_rn(acc[o] + __half2float(bias[o]));
}

// Image (B,3,H,W) NCHW fp16 / fp32 -> (B,4,H,W) fp16 with a zero fourth plane: the encoder's conv_in (3 -> C) then runs
// on the UNet's conv_in kernel (4 input channels) with a zero-padded weight.
__global__ void vae_image_pad_kernel(const void* __restrict__ x, int x_is_half, __half* __restrict__ out, int B, size_t HW) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t total = static_cast<size_t>(B) * 4 * HW;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t plane = i / HW;
    const int c = static_cast<int>(plane & 3);
    const size_t b = plane >> 2;
    __half v = __float2half(0.f);
    if (c < 3) {
      const size_t src = (b * 3 + c) * HW + (i - plane * HW);
      v = x_is_half ? reinterpret_cast<const __half*>(x)[src] : __float2half_rn(reinterpret_cast<const float*>(x)[src]);
    }
    out[i] = v;
  }
}

// Encoder tail: conv_out (3x3 pad 1, C -> 8 moments) on the GroupNorm+SiLU'ed NHWC input, quant_conv (1x1, 8 -> 8),
// DiagonalGaussianDistribution (mean | logvar, logvar clamped to [-30, 20], std = exp(logvar / 2)) and
// `latent_dist.sample() * scaling_factor` with the caller's noise draw. One warp per latent pixel. Rounding points of the
// fp16 module under the reference's torch.autocast (every `sample()` runs inside one): conv_out and quant_conv outputs
// and 0.5 * logvar are fp16; `exp` is on autocast's fp32 list, so std, std * noise, + mean and * scaling_factor are
// fp32 and the latent leaves as fp32.
__global__ void __launch_bounds__(256) vae_moments_sample_kernel(const __half* __restrict__ x, const __half* __restrict__ w,
                                                                 const __half* __restrict__ bias,
                                                                 const __half* __restrict__ wq,
                                                                 const __half* __restrict__ bq,
                                                                 const __half* __restrict__ noise, float scaling,
                                                                 float* __restrict__ out, int B, int H, int W, int C) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __half swm[];  // [8][9][C]
  for (int i = threadIdx.x * 8; i < 72 * C; i += blockDim.x * 8)
    *reinterpret_cast<uint4*>(swm + i) = *reinterpret_cast<const uint4*>(w + i);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int HW = H * W;
  const int pix = blockIdx.x * (blockDim.x >> 5) + warp;
  if (pix >= B * HW) return;
  const int b = pix / HW, r = pix - b * HW;
  const int h = r / W, xw = r - h * W;
  const int vpt = C >> 3;
  float acc[8];
#pragma unroll
  for (int o = 0; o < 8; ++o) acc[o] = 0.f;
  for (int v = lane; v < 9 * vpt; v += 32) {
    const int tap = v / vpt;
    const int c0 = (v - tap * vpt) * 8;
    const int hh = h + tap / 3 - 1, ww = xw + tap % 3 - 1;
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
    const uint4 ux = *reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(b) * H + hh) * W + ww) * C + c0);
    const __half2* hx = reinterpret_cast<const __half2*>(&ux);
#pragma unroll
    for (int o = 0; o < 8; ++o) {
      const uint4 uw = *reinterpret_cast<const uint4*>(swm + (o * 9 + tap) * C + c0);
      const __half2* hw = reinterpret_cast<const __half2*>(&uw);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 a = __half22float2(hx[i]), wf = __half22float2(hw[i]);
        acc[o] += a.x * wf.x + a.y * wf.y;
      }
    }
  }
#pragma unroll
  for (int o = 0; o < 8; ++o)
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], d);
  if (lane < 4) {
    float m[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) m[o] = rh(acc[o] + __half2float(bias[o]));
    float q_mean = __half2float(bq[lane]), q_logvar = __half2float(bq[4 + lane]);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      q_mean += __half2float(wq[lane * 8 + i]) * m[i];
      q_logvar += __half2float(wq[(4 + lane) * 8 + i]) * m[i];
    }
    const float mean = rh(q_mean);
    const float logvar = fminf(fmaxf(rh(q_logvar), -30.f), 20.f);
    const float stdv = expf(rh(0.5f * logvar));
    const size_t i = (static_cast<size_t>(b) * 4 + lane) * HW + r;
    const float nz = noise ? __half2float(noise[i]) : 0.f;
    out[i] = __fmul_rn(__fadd_rn(mean, __fmul_rn(stdv, nz)), scaling);
  }
}

}  // namespace

void run_vae_latent_prep(const void* z, int z_is_half, float scaling, const __half* w, const __half* bias, __half* out,
                         int B, int HW, cudaStream_t stream) {
  const int total = B * HW;
  launch_pdl(vae_latent_prep_kernel, dim3((total + 255) / 256), dim3(256), 0, stream, z, z_is_half, scaling, w, bias, out,
             B, HW);
}

void run_vae_row_softmax(__half* s, int rows, int n, float scale_log2e, cudaStream_t stream) {
  CFGPP_REQUIRE(n % 8 == 0, "softmax row length must be a multiple of 8");
  launch_pdl(vae_row_softmax_kernel, dim3(rows), dim3(256), 0, stream, s, n, scale_log2e);
}

void run_vae_conv_rgb(const __half* x, const __half* w, const __half* bias, __half* out, int B, int H, int W, int C,
                      cudaStream_t stream) {
  CFGPP_REQUIRE(C % 8 == 0 && 27 * C * 2 <= 48 * 1024, "conv_out: C % 8 == 0 and weights within 48 KB of shared memory");
  const size_t total = static_cast<size_t>(B) * H * W;
  launch_pdl(vae_conv_rgb_kernel, dim3(static_cast<unsigned>((total + 127) / 128)), dim3(128),
             static_cast<size_t>(27) * C * sizeof(__half), stream, x, w, bias, out, B, H, W, C);
}

}  // namespace cfgpp

namespace cfgpp {

void run_vae_image_pad(const void* x, int x_is_half, __half* out, int B, int H, int W, cudaStream_t stream) {
  const size_t HW = static_cast<size_t>(H) * W;
  const size_t total = static_cast<size_t>(B) * 4 * HW;
  const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, num_sms() * 32));
  launch_pdl(vae_image_pad_kernel, dim3(blocks), dim3(256), 0, stream, x, x_is_half, out, B, HW);
}

void run_vae_moments_sample(const __half* x, const __half* w, const __half* bias, const __half* wq, const __half* bq,
                            const __half* noise, float scaling, float* out, int B, int H, int W, int C,
                            cudaStream_t stream) {
  const size_t smem = static_cast<size_t>(72) * C * sizeof(__half);
  CFGPP_REQUIRE(C % 8 == 0 && smem <= 160 * 1024, "encoder conv_out: C % 8 == 0 and weights within 160 KB of shared memory");
  static bool configured = false;
  if (!configured) {
    CFGPP_CHECK_CUDA(cudaFuncSetAttribute(vae_moments_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    configured = true;
  }
  const int warps = 8;
  const int total = B * H * W;
  launch_pdl(vae_moments_sample_kernel, dim3((total + warps - 1) / warps), dim3(warps * 32), smem, stream, x, w, bias, wq, bq,
             noise, scaling, out, B, H, W, C);
}

}  // namespace cfgpp
