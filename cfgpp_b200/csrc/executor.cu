// cfgpp_b200 — weight store, device arena and stream-K workspace of the executors (see executor.cuh).
#include "executor.cuh"

#include <algorithm>

#include "../../include/cfgpp_b200.h"
#include "gemm.cuh"

namespace cfgpp {

namespace {

__global__ void f32_to_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = __float2half_rn(in[i]);
}

// (Cout, Cin, 3, 3) -> [Cout][tap][Cin]
__global__ void pack_conv3x3_kernel(const __half* __restrict__ in, __half* __restrict__ out, int Cout, int Cin) {
  const size_t n = static_cast<size_t>(Cout) * Cin * 9;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ci = i % Cin;
    const size_t t = i / Cin;
    const int tap = t % 9;
    const int co = t / 9;
    out[i] = in[(static_cast<size_t>(co) * Cin + ci) * 9 + tap];
  }
}

}  // namespace

int grid_for(size_t n) { return static_cast<int>(std::min<size_t>((n + 255) / 256, num_sms() * 8)); }

// ---- DeviceArena ----------------------------------------------------------------------------------------------------
void* DeviceArena::alloc(size_t bytes) {
  bytes = (bytes + 255) & ~static_cast<size_t>(255);
  ptrs_.reserve(ptrs_.size() + 1);  // the push_back below cannot throw once the allocation has succeeded
  void* p = nullptr;
  CFGPP_CHECK_CUDA(cudaMalloc(&p, std::max<size_t>(bytes, 256)));
  ptrs_.push_back(p);
  bytes_ += bytes;
  return p;
}

void DeviceArena::clear() {
  for (void* p : ptrs_) cudaFree(p);
  ptrs_.clear();
  bytes_ = 0;
}

// ---- WeightStore ----------------------------------------------------------------------------------------------------
size_t WeightStore::Weight::numel() const {
  size_t n = 1;
  for (auto d : shape) n *= static_cast<size_t>(d);
  return n;
}

void WeightStore::load(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype,
                       cudaStream_t stream) {
  CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "weight dtype must be fp16 or fp32");
  Weight w;
  w.shape.assign(shape, shape + ndim);
  const size_t n = w.numel();
  __half* p = nullptr;
  CFGPP_CHECK_CUDA(cudaMalloc(&p, std::max<size_t>(n, 8) * sizeof(__half)));
  w.data.reset(p);
  if (dtype == CFGPP_F16) {
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(p, data, n * sizeof(__half), cudaMemcpyDeviceToDevice, stream));
  } else {
    f32_to_f16_kernel<<<grid_for(n), 256, 0, stream>>>(static_cast<const float*>(data), p, n);
    CFGPP_CHECK_CUDA(cudaGetLastError());
  }
  raw_[key] = std::move(w);
}

const WeightStore::Weight& WeightStore::raw(const std::string& key) const {
  auto it = raw_.find(key);
  if (it == raw_.end()) throw Error(-10, "missing weight: " + key);
  return it->second;
}

__half* WeightStore::plain(const std::string& key, size_t expect_numel) const {
  const Weight& t = raw(key);
  if (t.numel() != expect_numel)
    throw Error(-11, "weight " + key + " has " + std::to_string(t.numel()) + " elements, expected " +
                         std::to_string(expect_numel));
  return t.p();
}

__half* WeightStore::packed_conv3x3(const std::string& key) {
  auto it = conv3x3_.find(key);
  if (it != conv3x3_.end()) return it->second;
  const Weight& t = raw(key);
  CFGPP_REQUIRE(t.shape.size() == 4 && t.shape[2] == 3 && t.shape[3] == 3, "expected (Cout,Cin,3,3): " + key);
  const int Cout = static_cast<int>(t.shape[0]), Cin = static_cast<int>(t.shape[1]);
  __half* out = alloc(t.numel());
  pack_conv3x3_kernel<<<grid_for(t.numel()), 256>>>(t.p(), out, Cout, Cin);
  CFGPP_CHECK_CUDA(cudaGetLastError());
  conv3x3_[key] = out;
  return out;
}

// ---- StreamKWorkspace -----------------------------------------------------------------------------------------------
StreamKWorkspace::StreamKWorkspace(int device) {
  CFGPP_CHECK_CUDA(cudaSetDevice(device));
  streamk_alloc(&ws_, &flags_);
}
StreamKWorkspace::~StreamKWorkspace() { streamk_free(ws_, flags_); }

}  // namespace cfgpp
