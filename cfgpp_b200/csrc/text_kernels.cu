// cfgpp_b200 — the small kernels of the CLIP text towers (see text_encoder.cuh): token + position embedding, the
// 77-token causal self-attention (one CTA per (head, prompt); K / V of a head live in shared memory, fp32 scores and
// probabilities — the sequences are far too short for a tensor-core tile), the MLP activation, and the gather of the
// pooled (<|endoftext|>) row. The projections and MLP GEMMs run on the wgmma GEMM of gemm.cu.
#include "common.cuh"
#include "text_encoder.cuh"

namespace cfgpp {

namespace {

// patch rows of an NCHW image: out[(b * g + py) * g + px][(c * P + ky) * P + kx] = fp16(x[b, c, py P + ky, px P + kx]),
// columns 3 P P .. Kp - 1 zero (g = S / P)
__global__ void clip_patchify_kernel(const void* __restrict__ x, int is_half, __half* __restrict__ out, int B, int S,
                                     int P, int Kp) {
  const int g = S / P, K = 3 * P * P;
  const size_t n = static_cast<size_t>(B) * g * g * Kp;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % Kp);
    const size_t row = i / Kp;
    __half v = __float2half(0.f);
    if (k < K) {
      const int px = static_cast<int>(row % g), py = static_cast<int>((row / g) % g), b = static_cast<int>(row / g / g);
      const int c = k / (P * P), ky = (k / P) % P, kx = k % P;
      const size_t src = ((static_cast<size_t>(b) * 3 + c) * S + py * P + ky) * S + px * P + kx;
      v = is_half ? static_cast<const __half*>(x)[src] : __float2half_rn(static_cast<const float*>(x)[src]);
    }
    out[i] = v;
  }
}

// x[b, 0, :] = fp16(cls + pos[0]), x[b, 1 + p, :] = fp16(pe[b np + p] + pos[1 + p])
__global__ void clip_vision_embed_kernel(const __half* __restrict__ pe, const __half* __restrict__ cls,
                                         const __half* __restrict__ pos, __half* __restrict__ out, int B, int np,
                                         int D) {
  const int T = np + 1;
  const size_t n = static_cast<size_t>(B) * T * D;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(i % D);
    const int t = static_cast<int>((i / D) % T);
    const int b = static_cast<int>(i / D / T);
    const __half a = t == 0 ? cls[d] : pe[(static_cast<size_t>(b) * np + t - 1) * D + d];
    out[i] = __float2half_rn(__half2float(a) + __half2float(pos[static_cast<size_t>(t) * D + d]));
  }
}

// out[r, :] = fp16(tok[ids[r], :] + pos[r % T, :])   (one rounding, as the fp16 module's `inputs_embeds + position_embeddings`)
__global__ void clip_embed_kernel(const int* __restrict__ ids, const uint4* __restrict__ tok, const uint4* __restrict__ pos,
                                  uint4* __restrict__ out, int M, int T, int Dv, int vocab) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t total = static_cast<size_t>(M) * Dv;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / Dv), c = static_cast<int>(i - static_cast<size_t>(r) * Dv);
    int id = ids[r];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);  // ids are validated on the host; never read out of bounds
    const uint4 a = tok[static_cast<size_t>(id) * Dv + c];
    const uint4 b = pos[static_cast<size_t>(r % T) * Dv + c];
    uint4 o;
    const __half2* ha = reinterpret_cast<const __half2*>(&a);
    const __half2* hb = reinterpret_cast<const __half2*>(&b);
    __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) ho[k] = __hadd2(ha[k], hb[k]);
    out[i] = o;
  }
}

// Causal self-attention of one (head, prompt): qkv [B*T][3*D] (q | k | v column blocks, head h at columns h*64..),
// out [B*T][D]. softmax(q k^T * scale + causal mask) v with fp32 scores / probabilities / accumulation and one
// rounding of the output. No padding mask: the reference passes none (latent_sdxl.py:85, latent_diffusion.py:105).
constexpr int kClipHD = 64;
constexpr int kClipMaxT = 128;
__global__ void __launch_bounds__(128) clip_attn_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int T,
                                                        int D, float scale) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ __half ks[kClipMaxT][kClipHD + 2];  // +2: rows 33 words apart -> lanes reading one column hit 32 banks
  __shared__ __half vs[kClipMaxT][kClipHD];
  __shared__ float qs[4][kClipHD];
  __shared__ float ps[4][kClipMaxT];
  const int h = blockIdx.x, b = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t ld = static_cast<size_t>(3) * D;
  const __half* base = qkv + static_cast<size_t>(b) * T * ld + static_cast<size_t>(h) * kClipHD;
  for (int i = threadIdx.x; i < T * (kClipHD / 2); i += blockDim.x) {
    const int t = i / (kClipHD / 2), c = (i - t * (kClipHD / 2)) * 2;
    *reinterpret_cast<__half2*>(&ks[t][c]) = *reinterpret_cast<const __half2*>(base + t * ld + D + c);
    *reinterpret_cast<__half2*>(&vs[t][c]) = *reinterpret_cast<const __half2*>(base + t * ld + 2 * D + c);
  }
  __syncthreads();
  for (int i = warp; i < T; i += 4) {
    {
      const float2 q2 = __half22float2(*reinterpret_cast<const __half2*>(base + i * ld + lane * 2));
      qs[warp][lane * 2] = q2.x;
      qs[warp][lane * 2 + 1] = q2.y;
    }
    __syncwarp();
    float s[kClipMaxT / 32];
    float mx = -INFINITY;
#pragma unroll
    for (int u = 0; u < kClipMaxT / 32; ++u) {
      const int j = lane + u * 32;
      s[u] = -INFINITY;
      if (j <= i) {
        float acc = 0.f;
#pragma unroll 8
        for (int d = 0; d < kClipHD; d += 2) {
          const float2 k2 = __half22float2(*reinterpret_cast<const __half2*>(&ks[j][d]));
          acc = fmaf(qs[warp][d], k2.x, acc);
          acc = fmaf(qs[warp][d + 1], k2.y, acc);
        }
        s[u] = acc * scale;
      }
      mx = fmaxf(mx, s[u]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int u = 0; u < kClipMaxT / 32; ++u) {
      const int j = lane + u * 32;
      if (j <= i) {
        const float p = __expf(s[u] - mx);
        ps[warp][j] = p;
        sum += p;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __syncwarp();
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j <= i; ++j) {
      const float p = ps[warp][j];
      const float2 v2 = __half22float2(*reinterpret_cast<const __half2*>(&vs[j][lane * 2]));
      o0 = fmaf(p, v2.x, o0);
      o1 = fmaf(p, v2.y, o1);
    }
    const float inv = 1.f / sum;
    *reinterpret_cast<__half2*>(out + (static_cast<size_t>(b) * T + i) * D + static_cast<size_t>(h) * kClipHD + lane * 2) =
        __floats2half2_rn(o0 * inv, o1 * inv);
    __syncwarp();  // qs / ps of this warp are rewritten by the next row
  }
}

// quick_gelu as transformers' QuickGELUActivation runs it on an fp16 module, `x * torch.sigmoid(1.702 * x)`: three fp16
// tensor ops, each computed in fp32 and rounded to fp16 (torch's sigmoid is 1 / (1 + exp(-a)) with the precise expf).
CFGPP_DEVICE float quick_gelu_f16(float x) {
  const float a = __half2float(__float2half_rn(1.702f * x));
  const float s = __half2float(__float2half_rn(1.f / (1.f + expf(-a))));
  return x * s;  // exact in fp32 (two 11-bit significands); the caller's rounding is the third fp16 op
}

// In-place MLP activation on fp16: 0 = quick_gelu x * sigmoid(1.702 x) (OpenAI CLIP), 1 = gelu (erf; OpenCLIP bigG)
__global__ void clip_act_kernel(uint4* __restrict__ x, size_t nvec, int mode) {
  pdl_launch_dependents();
  pdl_wait();
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    uint4 v = x[i];
    __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 f = __half22float2(h[k]);
      if (mode == 0) {
        f.x = quick_gelu_f16(f.x);
        f.y = quick_gelu_f16(f.y);
      } else {
        f.x = 0.5f * f.x * (1.f + erff(f.x * 0.70710678118654752f));
        f.y = 0.5f * f.y * (1.f + erff(f.y * 0.70710678118654752f));
      }
      h[k] = __floats2half2_rn(f.x, f.y);
    }
    x[i] = v;
  }
}

// out[b, :] = x[b * T + index[b], :]
__global__ void clip_gather_rows_kernel(const uint4* __restrict__ x, const int* __restrict__ index, uint4* __restrict__ out,
                                        int B, int T, int Dv) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Dv) return;
  const int b = i / Dv, c = i - b * Dv;
  int t = index[b];
  t = t < 0 ? 0 : (t >= T ? T - 1 : t);
  out[i] = x[(static_cast<size_t>(b) * T + t) * Dv + c];
}

}  // namespace

void run_clip_embed(const int* ids, const __half* tok, const __half* pos, __half* out, int M, int T, int D, int vocab,
                    cudaStream_t stream) {
  CFGPP_REQUIRE(D % 8 == 0, "hidden size must be a multiple of 8");
  const size_t total = static_cast<size_t>(M) * (D / 8);
  const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, 4096));
  launch_pdl(clip_embed_kernel, dim3(blocks), dim3(256), 0, stream, ids, reinterpret_cast<const uint4*>(tok),
             reinterpret_cast<const uint4*>(pos), reinterpret_cast<uint4*>(out), M, T, D / 8, vocab);
}

void run_clip_attention(const __half* qkv, __half* out, int B, int T, int heads, int D, cudaStream_t stream) {
  CFGPP_REQUIRE(D == heads * kClipHD, "the CLIP text towers use 64-wide heads");
  CFGPP_REQUIRE(T >= 1 && T <= kClipMaxT, "at most 128 tokens per prompt");
  launch_pdl(clip_attn_kernel, dim3(heads, B), dim3(128), 0, stream, qkv, out, T, D, 1.0f / sqrtf(static_cast<float>(kClipHD)));
}

void run_clip_activation(__half* x, size_t n, int mode, cudaStream_t stream) {
  CFGPP_REQUIRE(n % 8 == 0, "activation size must be a multiple of 8");
  CFGPP_REQUIRE(mode == 0 || mode == 1, "hidden_act: 0 quick_gelu, 1 gelu");
  const size_t nvec = n / 8;
  const int blocks = static_cast<int>(std::min<size_t>((nvec + 255) / 256, 4096));
  launch_pdl(clip_act_kernel, dim3(blocks), dim3(256), 0, stream, reinterpret_cast<uint4*>(x), nvec, mode);
}

void run_clip_gather_rows(const __half* x, const int* index, __half* out, int B, int T, int D, cudaStream_t stream) {
  const int total = B * (D / 8);
  launch_pdl(clip_gather_rows_kernel, dim3((total + 127) / 128), dim3(128), 0, stream, reinterpret_cast<const uint4*>(x),
             index, reinterpret_cast<uint4*>(out), B, T, D / 8);
}

void run_clip_patchify(const void* image, int is_half, __half* out, int B, int S, int P, int Kp, cudaStream_t stream) {
  const size_t n = static_cast<size_t>(B) * (S / P) * (S / P) * Kp;
  clip_patchify_kernel<<<static_cast<int>(std::min<size_t>((n + 255) / 256, 8192)), 256, 0, stream>>>(image, is_half, out,
                                                                                                       B, S, P, Kp);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

void run_clip_vision_embed(const __half* pe, const __half* cls, const __half* pos, __half* out, int B, int np, int D,
                           cudaStream_t stream) {
  const size_t n = static_cast<size_t>(B) * (np + 1) * D;
  clip_vision_embed_kernel<<<static_cast<int>(std::min<size_t>((n + 255) / 256, 8192)), 256, 0, stream>>>(pe, cls, pos,
                                                                                                           out, B, np, D);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

}  // namespace cfgpp
