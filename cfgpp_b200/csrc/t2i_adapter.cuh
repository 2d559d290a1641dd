// cfgpp_b200 — T2I-Adapter executor (diffusers 0.27.1 `T2IAdapter` with `FullAdapter` / `FullAdapterXL`): the small CNN
// that turns a conditioning image into the four feature maps a UNet handle adds into its down path
// (cfgpp_t2i_attach). It runs once per image, not per step:
//   PixelUnshuffle(f) -> conv_in 3x3 -> 4 AdapterBlocks, each [AvgPool2d(2) if down] -> [in_conv 1x1 if the channel
//   count changes] -> num_res_blocks x (h = block2_1x1(relu(block1_3x3(x))); x = h + x); every block's output is one
//   feature, multiplied by the conditioning scale in fp16.
// Activations are NHWC fp16. The convolutions are the UNet's wgmma GEMMs (make_conv3x3_op / make_linear_op, block2's
// residual add in the epilogue: fp16(fp16(acc + bias) + x)); pixel unshuffle, the 2x2 average pool, ReLU and the scale
// are the small kernels of t2i_adapter.cu.
#pragma once
#include <functional>
#include <string>
#include <vector>

#include "../../include/cfgpp_b200.h"
#include "executor.cuh"
#include "gemm.cuh"
#include "ops.cuh"

namespace cfgpp {

class T2IAdapter {
 public:
  static constexpr int kFeatures = 4;
  T2IAdapter(const cfgpp_t2i_adapter_desc& d, int device);
  void load_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                   cudaStream_t stream);
  void finalize_weights(cudaStream_t stream);
  // image (batch, in_channels, H, W) NCHW fp16 / fp32 in [0, 1] -> features[k] NHWC fp16 (batch, h_k, w_k, C_k),
  // already multiplied by `scale`. H and W must be multiples of total_factor().
  void forward(const void* image, int dtype, int batch, int H, int W, float scale, __half* const* features,
               cudaStream_t stream);
  int total_factor() const;
  double flops() const { return plan_.flops; }
  size_t workspace_bytes() const { return plan_.arena.bytes(); }

 private:
  struct Block {
    int cin, cout;
    bool down;
  };
  Block block(int i) const;
  void expect_shape(const std::string& key, std::vector<int64_t> shape) const;
  void prepare(int batch, int H, int W);
  void add(std::function<void(cudaStream_t)> fn) { plan_.steps.push_back(std::move(fn)); }
  void add_gemm(const GemmOp& op) {
    plan_.flops += op.flops();
    plan_.steps.push_back([op](cudaStream_t st) { run_gemm_op(op, st); });
  }

  cfgpp_t2i_adapter_desc d_;
  int device_;
  bool finalized_ = false;
  WeightStore weights_;
  StreamKWorkspace sk_;
  struct Plan {
    std::vector<std::function<void(cudaStream_t)>> steps;
    double flops = 0.0;
    DeviceArena arena;
    int batch = 0, h = 0, w = 0;  // batch 0: nothing prepared
  } plan_;
  // set per forward() call, read by the plan's steps when they are enqueued
  const void* image_ = nullptr;
  int image_half_ = 0;
  float scale_ = 1.0f;
  __half* out_[kFeatures] = {};
};

}  // namespace cfgpp
