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
  conv3x3_[key] = alloc(t.numel());
  refresh_conv3x3(key, nullptr);
  return conv3x3_[key];
}

size_t WeightStore::refresh_conv3x3(const std::string& key, cudaStream_t stream) {
  auto it = conv3x3_.find(key);
  if (it == conv3x3_.end()) return 0;
  const Weight& t = raw(key);
  pack_conv3x3_kernel<<<grid_for(t.numel()), 256, 0, stream>>>(t.p(), it->second, static_cast<int>(t.shape[0]),
                                                               static_cast<int>(t.shape[1]));
  CFGPP_CHECK_CUDA(cudaGetLastError());
  return 2 * t.numel() * sizeof(__half);
}

// ---- LoRA ----------------------------------------------------------------------------------------------------
namespace {

WeightStore::Weight::Ptr device_halves(size_t n) {
  __half* p = nullptr;
  CFGPP_CHECK_CUDA(cudaMalloc(&p, std::max<size_t>(n, 8) * sizeof(__half)));
  return WeightStore::Weight::Ptr(p);
}

}  // namespace

void WeightStore::lora_add(int adapter, const std::string& key, const void* down, const void* up, int rank, float alpha,
                           int dtype, cudaStream_t stream) {
  CFGPP_REQUIRE(dtype == CFGPP_F16 || dtype == CFGPP_F32, "LoRA factor dtype must be fp16 or fp32");
  CFGPP_REQUIRE(adapter >= 0 && adapter < 64, "adapter id must be 0..63");
  CFGPP_REQUIRE(down && up, "null LoRA factor for " + key);
  const Weight& w = raw(key);
  CFGPP_REQUIRE(w.shape.size() >= 2, "a LoRA targets a weight of 2 or more dimensions: " + key);
  CFGPP_REQUIRE(rank >= 1 && rank <= kMaxLoraRank, "LoRA rank must be 1..128: " + key);
  auto it = lora_.find(key);
  if (it != lora_.end()) {
    for (const LoraFactor& f : it->second.factors)
      if (f.adapter == adapter) throw Error(-12, "adapter " + std::to_string(adapter) + " already targets " + key);
    if (static_cast<int>(it->second.factors.size()) >= kMaxLoraPerTarget)
      throw Error(-12, "too many LoRA adapters on " + key + " (at most 4 per weight)");
  }
  const size_t N = static_cast<size_t>(w.shape[0]), K = w.numel() / N;
  auto ingest = [&](const void* src, size_t n) {
    Weight::Ptr dst = device_halves(n);
    if (dtype == CFGPP_F16) {
      CFGPP_CHECK_CUDA(cudaMemcpyAsync(dst.get(), src, n * sizeof(__half), cudaMemcpyDeviceToDevice, stream));
    } else {
      f32_to_f16_kernel<<<grid_for(n), 256, 0, stream>>>(static_cast<const float*>(src), dst.get(), n);
      CFGPP_CHECK_CUDA(cudaGetLastError());
    }
    return dst;
  };
  LoraFactor f{adapter, rank, alpha, ingest(down, rank * K), ingest(up, N * rank)};
  if (it == lora_.end()) {  // first adapter on this key: raw storage still holds the base weight
    LoraTarget t;
    t.backup = device_halves(w.numel());
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(t.backup.get(), w.p(), w.numel() * sizeof(__half), cudaMemcpyDeviceToDevice, stream));
    it = lora_.emplace(key, std::move(t)).first;
  }
  it->second.factors.push_back(std::move(f));
  lora_adapters_ = std::max(lora_adapters_, adapter + 1);
}

std::set<std::string> WeightStore::lora_apply(const float* scales, int n, cudaStream_t stream, size_t* bytes) {
  CFGPP_REQUIRE(n == lora_adapters_ && (n == 0 || scales), "one scale per adapter id (" + std::to_string(lora_adapters_) + ")");
  std::set<std::string> touched;
  for (auto& kv : lora_) {
    const Weight& w = raw(kv.first);
    const int N = static_cast<int>(w.shape[0]), K = static_cast<int>(w.numel() / N);
    LoraMergeArgs a{};
    for (const LoraFactor& f : kv.second.factors) {
      a.down[a.n] = f.down.get();
      a.up[a.n] = f.up.get();
      a.rank[a.n] = f.rank;
      a.coef[a.n] = scales[f.adapter] * f.alpha / static_cast<float>(f.rank);
      *bytes += (static_cast<size_t>(N) + K) * f.rank * sizeof(__half);
      ++a.n;
    }
    run_lora_merge(kv.second.backup.get(), a, N, K, w.p(), stream);
    *bytes += 2 * w.numel() * sizeof(__half);
    touched.insert(kv.first);
  }
  return touched;
}

std::set<std::string> WeightStore::lora_restore(cudaStream_t stream, size_t* bytes) {
  std::set<std::string> touched;
  for (auto& kv : lora_) {
    const Weight& w = raw(kv.first);
    CFGPP_CHECK_CUDA(cudaMemcpyAsync(w.p(), kv.second.backup.get(), w.numel() * sizeof(__half), cudaMemcpyDeviceToDevice, stream));
    *bytes += 2 * w.numel() * sizeof(__half);
    touched.insert(kv.first);
  }
  return touched;
}

void WeightStore::lora_free(cudaStream_t stream) {
  CFGPP_CHECK_CUDA(cudaStreamSynchronize(stream));  // the restore and the repacks still read what is freed here
  lora_.clear();
  lora_adapters_ = 0;
}

size_t WeightStore::lora_backup_bytes() const {
  size_t b = 0;
  for (auto& kv : lora_) b += raw(kv.first).numel() * sizeof(__half);
  return b;
}

// ---- StreamKWorkspace -----------------------------------------------------------------------------------------------
StreamKWorkspace::StreamKWorkspace(int device) {
  CFGPP_CHECK_CUDA(cudaSetDevice(device));
  streamk_alloc(&ws_, &flags_);
}
StreamKWorkspace::~StreamKWorkspace() { streamk_free(ws_, flags_); }

}  // namespace cfgpp
