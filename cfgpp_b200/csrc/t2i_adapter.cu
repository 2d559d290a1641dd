// cfgpp_b200 — T2I-Adapter: its small kernels (pixel unshuffle, 2x2 average pool, ReLU, scale), the gated add the UNet
// step graph runs per feature, and the adapter executor (see t2i_adapter.cuh).
#include "t2i_adapter.cuh"

#include <algorithm>

#include "common.cuh"

namespace cfgpp {

void gemm_configure();

namespace {

__global__ void pixel_unshuffle_kernel(const void* __restrict__ x, int x_is_half, __half* __restrict__ out, int B,
                                       int C, int H, int W, int f) {
  const int Ho = H / f, Wo = W / f, Co = C * f * f;
  const size_t n = static_cast<size_t>(B) * Ho * Wo * Co;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int co = i % Co;
    size_t t = i / Co;
    const int xo = t % Wo;
    t /= Wo;
    const int yo = t % Ho;
    const size_t b = t / Ho;
    const int c = co / (f * f), ij = co % (f * f);
    const size_t src = ((b * C + c) * H + static_cast<size_t>(yo) * f + ij / f) * W + static_cast<size_t>(xo) * f + ij % f;
    out[i] = x_is_half ? reinterpret_cast<const __half*>(x)[src] : __float2half_rn(reinterpret_cast<const float*>(x)[src]);
  }
}

// 8 channels per thread; torch's avg_pool2d sums the window row by row from 0 in fp32 and divides by 4
__global__ void avgpool2x2_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int H, int W, int Cv) {
  const int Ho = H / 2, Wo = W / 2;
  const size_t n = static_cast<size_t>(B) * Ho * Wo * Cv;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = i % Cv;
    size_t t = i / Cv;
    const int xo = t % Wo;
    t /= Wo;
    const int yo = t % Ho;
    const size_t b = t / Ho;
    const size_t r0 = ((b * H + 2 * yo) * W + 2 * xo) * Cv + cv, r1 = r0 + static_cast<size_t>(W) * Cv;
    const uint4 v[4] = {x[r0], x[r0 + Cv], x[r1], x[r1 + Cv]};
    uint4 o;
    __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 s = make_float2(0.f, 0.f);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = __half22float2(reinterpret_cast<const __half2*>(&v[q])[k]);
        s.x += f.x;
        s.y += f.y;
      }
      ho[k] = __floats2half2_rn(s.x / 4.0f, s.y / 4.0f);
    }
    out[i] = o;
  }
}

__global__ void relu_kernel(__half* __restrict__ x, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const __half v = x[i];
    x[i] = __hgt(v, __float2half(0.f)) ? v : __float2half(0.f);
  }
}

__global__ void scale_kernel(const __half* x, float s, __half* out, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = __float2half_rn(__half2float(x[i]) * s);
}

// A launch of the step graph: PDL like its neighbours. The word is read after pdl_wait (select_step wrote it).
__global__ void t2i_add_kernel(uint4* __restrict__ h, const uint4* __restrict__ feat, int NB, int B, size_t per_image_v,
                               const int* __restrict__ on) {
  pdl_launch_dependents();
  pdl_wait();
  if (*on == 0) return;
  const size_t n = static_cast<size_t>(NB) * per_image_v;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t img = i / per_image_v, off = i - img * per_image_v;
    uint4 a = h[i];
    const uint4 f = feat[(img % B) * per_image_v + off];
    __half2* ha = reinterpret_cast<__half2*>(&a);
    const __half2* hf = reinterpret_cast<const __half2*>(&f);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 x = __half22float2(ha[k]), y = __half22float2(hf[k]);
      ha[k] = __floats2half2_rn(x.x + y.x, x.y + y.y);
    }
    h[i] = a;
  }
}

}  // namespace

void run_pixel_unshuffle(const void* x, int x_is_half, __half* out, int B, int C, int H, int W, int f,
                         cudaStream_t stream) {
  CFGPP_REQUIRE(f >= 1 && H % f == 0 && W % f == 0, "pixel unshuffle: H and W must be multiples of the factor");
  const size_t n = static_cast<size_t>(B) * H * W * C;
  pixel_unshuffle_kernel<<<grid_for(n), 256, 0, stream>>>(x, x_is_half, out, B, C, H, W, f);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

void run_avgpool2x2(const __half* x, __half* out, int B, int H, int W, int C, cudaStream_t stream) {
  CFGPP_REQUIRE(H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "average pool: even H, W and C % 8 == 0");
  const size_t n = static_cast<size_t>(B) * (H / 2) * (W / 2) * (C / 8);
  avgpool2x2_kernel<<<grid_for(n), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out),
                                                     B, H, W, C / 8);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

void run_relu(__half* x, size_t n, cudaStream_t stream) {
  relu_kernel<<<grid_for(n), 256, 0, stream>>>(x, n);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

void run_scale(const __half* x, float s, __half* out, size_t n, cudaStream_t stream) {
  scale_kernel<<<grid_for(n), 256, 0, stream>>>(x, s, out, n);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

void run_t2i_add(__half* h, const __half* feat, int NB, int B, size_t per_image, const int* on, cudaStream_t stream) {
  CFGPP_REQUIRE(per_image % 8 == 0 && B >= 1 && NB >= B, "T2I add: per-image size % 8 and NB >= B");
  const size_t n = static_cast<size_t>(NB) * (per_image / 8);
  launch_pdl(t2i_add_kernel, dim3(grid_for(n)), dim3(256), 0, stream, reinterpret_cast<uint4*>(h),
             reinterpret_cast<const uint4*>(feat), NB, B, per_image / 8, on);
}

// ------------------------------------------------------------------------------------------------------------
// executor
// ------------------------------------------------------------------------------------------------------------
T2IAdapter::T2IAdapter(const cfgpp_t2i_adapter_desc& d, int device) : d_(d), device_(device), sk_(device) {
  CFGPP_CHECK_CUDA(cudaSetDevice(device));
  CFGPP_REQUIRE(d.kind == 0 || d.kind == 1, "T2I-Adapter kind must be 0 (full_adapter) or 1 (full_adapter_xl)");
  CFGPP_REQUIRE(d.in_channels == 1 || d.in_channels == 3, "T2I-Adapter in_channels must be 1 or 3");
  CFGPP_REQUIRE(d.downscale_factor >= 1 && d.downscale_factor <= 16, "T2I-Adapter downscale_factor must be 1..16");
  CFGPP_REQUIRE(d.in_channels * d.downscale_factor * d.downscale_factor % 64 == 0,
                "in_channels * downscale_factor^2 must be a multiple of 64 (the convolution's K block)");
  CFGPP_REQUIRE(d.num_res_blocks >= 1 && d.num_res_blocks <= 8, "T2I-Adapter num_res_blocks must be 1..8");
  for (int i = 0; i < kFeatures; ++i)
    CFGPP_REQUIRE(d.channels[i] >= 64 && d.channels[i] % 64 == 0, "T2I-Adapter channels must be multiples of 64");
  CFGPP_REQUIRE(d.kind == 0 || d.channels[2] == d.channels[3],
                "full_adapter_xl: channels[3] must equal channels[2] (its last block keeps the width)");
  gemm_configure();
}

// diffusers FullAdapter: (c0,c0), (c[i-1],c[i],down); FullAdapterXL: (c0,c0), (c0,c1), (c1,c2,down), (c3,c3)
T2IAdapter::Block T2IAdapter::block(int i) const {
  const int* c = d_.channels;
  if (i == 0) return {c[0], c[0], false};
  if (d_.kind == 0) return {c[i - 1], c[i], true};
  if (i == 1) return {c[0], c[1], false};
  if (i == 2) return {c[1], c[2], true};
  return {c[3], c[3], false};
}

int T2IAdapter::total_factor() const { return d_.downscale_factor * (d_.kind == 0 ? 8 : 2); }

void T2IAdapter::load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                             cudaStream_t stream) {
  CFGPP_REQUIRE(!finalized_, "weights already finalized");
  weights_.load(key, data, shape, ndim, dtype, stream);
}

void T2IAdapter::expect_shape(const std::string& key, std::vector<int64_t> shape) const {
  CFGPP_REQUIRE(weights_.raw(key).shape == shape, "unexpected shape of " + key);
}

void T2IAdapter::finalize_weights(cudaStream_t stream) {
  CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));
  const int64_t cu = static_cast<int64_t>(d_.in_channels) * d_.downscale_factor * d_.downscale_factor;
  expect_shape("adapter.conv_in.weight", {d_.channels[0], cu, 3, 3});
  expect_shape("adapter.conv_in.bias", {d_.channels[0]});
  for (int i = 0; i < kFeatures; ++i) {
    const Block b = block(i);
    const std::string p = "adapter.body." + std::to_string(i);
    if (b.cin != b.cout) {
      expect_shape(p + ".in_conv.weight", {b.cout, b.cin, 1, 1});
      expect_shape(p + ".in_conv.bias", {b.cout});
    }
    for (int j = 0; j < d_.num_res_blocks; ++j) {
      const std::string r = p + ".resnets." + std::to_string(j);
      expect_shape(r + ".block1.weight", {b.cout, b.cout, 3, 3});
      expect_shape(r + ".block1.bias", {b.cout});
      expect_shape(r + ".block2.weight", {b.cout, b.cout, 1, 1});
      expect_shape(r + ".block2.bias", {b.cout});
    }
  }
  finalized_ = true;
  try {  // packs every 3x3 convolution
    prepare(1, total_factor(), total_factor());
  } catch (...) {
    finalized_ = false;
    throw;
  }
}

void T2IAdapter::prepare(int batch, int H, int W) {
  CFGPP_CHECK_CUDA(cudaSetDevice(device_));
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());  // a forward in flight may still use the old plan's workspace
  StreamKScope sk_scope(sk_.ws(), sk_.flags());  // the adapter's GEMM ops use its own stream-K workspace
  plan_.steps.clear();
  plan_.arena.clear();
  plan_.flops = 0.0;
  plan_.batch = 0;
  const int f = d_.downscale_factor, Ci = d_.in_channels, Cu = Ci * f * f;
  int h = H / f, w = W / f, C = d_.channels[0];
  const size_t px0 = static_cast<size_t>(batch) * h * w;
  const int cmax = *std::max_element(d_.channels, d_.channels + kFeatures);
  __half* x0 = plan_.arena.alloc<__half>(px0 * Cu);
  __half* t = plan_.arena.alloc<__half>(px0 * cmax);  // block1 output, ReLU'd in place
  __half* cur = plan_.arena.alloc<__half>(px0 * C);
  add([this, x0, batch, Ci, H, W, f](cudaStream_t st) {
    run_pixel_unshuffle(image_, image_half_, x0, batch, Ci, H, W, f, st);
  });
  add_gemm(make_conv3x3_op(x0, batch, h, w, Cu, weights_.packed_conv3x3("adapter.conv_in.weight"), C,
                           weights_.plain("adapter.conv_in.bias"), nullptr, 0, 1, cur));
  for (int i = 0; i < kFeatures; ++i) {
    const Block b = block(i);
    const std::string p = "adapter.body." + std::to_string(i);
    if (b.down) {
      __half* y = plan_.arena.alloc<__half>(static_cast<size_t>(batch) * (h / 2) * (w / 2) * C);
      const __half* xp = cur;
      add([=](cudaStream_t st) { run_avgpool2x2(xp, y, batch, h, w, C, st); });
      h /= 2;
      w /= 2;
      cur = y;
    }
    const int M = batch * h * w;
    if (b.cin != b.cout) {
      __half* y = plan_.arena.alloc<__half>(static_cast<size_t>(M) * b.cout);
      add_gemm(make_linear_op(cur, C, nullptr, 0, 0, weights_.plain(p + ".in_conv.weight"), M, b.cout, C,
                              weights_.plain(p + ".in_conv.bias"), nullptr, 0, 1, y, b.cout, false));
      cur = y;
      C = b.cout;
    }
    // the residual add writes x in place: a feature's scaled copy is taken before the next block reads x again
    for (int j = 0; j < d_.num_res_blocks; ++j) {
      const std::string r = p + ".resnets." + std::to_string(j);
      add_gemm(make_conv3x3_op(cur, batch, h, w, C, weights_.packed_conv3x3(r + ".block1.weight"), C,
                               weights_.plain(r + ".block1.bias"), nullptr, 0, 1, t));
      const size_t n = static_cast<size_t>(M) * C;
      add([=](cudaStream_t st) { run_relu(t, n, st); });
      add_gemm(make_linear_op(t, C, nullptr, 0, 0, weights_.plain(r + ".block2.weight"), M, C, C,
                              weights_.plain(r + ".block2.bias"), cur, C, 1, cur, C, false));
    }
    const __half* xp = cur;
    const size_t n = static_cast<size_t>(M) * C;
    add([this, xp, n, i](cudaStream_t st) { run_scale(xp, scale_, out_[i], n, st); });
  }
  CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
  plan_.batch = batch;
  plan_.h = H;
  plan_.w = W;
}

void T2IAdapter::forward(const void* image, int dtype, int batch, int H, int W, float scale, __half* const* features,
                         cudaStream_t stream) {
  CFGPP_REQUIRE(finalized_, "call cfgpp_t2i_adapter_finalize_weights first");
  CFGPP_REQUIRE(image != nullptr && features != nullptr, "null argument");
  CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "adapter image: fp16 or fp32 tensor");
  CFGPP_REQUIRE(batch >= 1 && batch <= 8, "adapter batch must be 1..8");
  const int tf = total_factor();
  CFGPP_REQUIRE(H >= tf && W >= tf && H % tf == 0 && W % tf == 0,
                "adapter image height and width must be multiples of " + std::to_string(tf));
  for (int k = 0; k < kFeatures; ++k) CFGPP_REQUIRE(features[k] != nullptr, "null feature buffer");
  if (batch != plan_.batch || H != plan_.h || W != plan_.w) prepare(batch, H, W);
  image_ = image;
  image_half_ = dtype == CFGPP_F16 ? 1 : 0;
  scale_ = scale;
  for (int k = 0; k < kFeatures; ++k) out_[k] = features[k];
  for (auto& fn : plan_.steps) fn(stream);
}

}  // namespace cfgpp
