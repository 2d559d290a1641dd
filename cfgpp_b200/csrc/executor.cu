// cfgpp_b200 — weight store, device arena and stream-K workspace of the executors (see executor.cuh).
#include "executor.cuh"

#include <algorithm>

#include "../../include/cfgpp_b200.h"
#include "gemm.cuh"
#include "ops.cuh"

namespace cfgpp {

namespace {

__global__ void f32_to_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = __float2half_rn(in[i]);
}

// (Cout, Cin, 3, 3) -> [Cout_p][tap][Cin_p], zero beyond Cout / Cin
__global__ void pack_conv3x3_kernel(const __half* __restrict__ in, __half* __restrict__ out, int Cout, int Cin,
                                    int Cout_p, int Cin_p) {
  const size_t n = static_cast<size_t>(Cout_p) * 9 * Cin_p;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ci = i % Cin_p;
    const size_t t = i / Cin_p;
    const int tap = t % 9;
    const int co = t / 9;
    out[i] = (co < Cout && ci < Cin) ? in[(static_cast<size_t>(co) * Cin + ci) * 9 + tap] : __float2half(0.f);
  }
}

// GEGLU proj rows (2*inner, K): per 128 rows interleave value / gate halves into 256-row tiles
__global__ void pack_geglu_kernel(const __half* __restrict__ in, __half* __restrict__ out, int inner, int K) {
  const size_t n = static_cast<size_t>(2) * inner * K;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int k = i % K;
    const int r = i / K;  // packed row
    const int tile = r / 256, w = r % 256;
    const int src_row = (w < 128) ? (tile * 128 + w) : (inner + tile * 128 + (w - 128));
    out[i] = in[static_cast<size_t>(src_row) * K + k];
  }
}

struct HeadMats {
  const __half* p[3];
};

// rows of `nmat` stacked (heads*hd, K) matrices -> [(mat, head, hdp)][K], rows hd..hdp-1 of every head zero
__global__ void pack_heads_rows_kernel(HeadMats mats, __half* __restrict__ out, int nmat, int heads, int hd, int hdp,
                                       int K) {
  const size_t n = static_cast<size_t>(nmat) * heads * hdp * K;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int k = i % K;
    size_t t = i / K;
    const int r = t % hdp;
    t /= hdp;
    const int h = t % heads;
    const int m = t / heads;
    out[i] = (r < hd) ? mats.p[m][(static_cast<size_t>(h) * hd + r) * K + k] : __float2half(0.f);
  }
}

// (N, heads*hd) -> (N, heads*hdp) with zero columns hd..hdp-1 per head
__global__ void pack_heads_cols_kernel(const __half* __restrict__ in, __half* __restrict__ out, int N, int heads, int hd,
                                       int hdp) {
  const size_t n = static_cast<size_t>(N) * heads * hdp;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = i % hdp;
    size_t t = i / hdp;
    const int h = t % heads;
    const int row = t / heads;
    out[i] = (c < hd) ? in[(static_cast<size_t>(row) * heads + h) * hd + c] : __float2half(0.f);
  }
}

std::string joined(const std::string& kind, const std::vector<std::string>& keys) {
  std::string name = kind + ":";
  for (auto& k : keys) name += k + "|";
  return name;
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

__half* WeightStore::packed(const std::string& name, Recipe r) {
  auto it = packed_.find(name);
  if (it != packed_.end()) return it->second.out;
  r.out = arena_.alloc<__half>(r.numel);
  run(r, nullptr);
  return packed_.emplace(name, std::move(r)).first->second.out;
}

size_t WeightStore::run(const Recipe& r, cudaStream_t stream) {
  const Weight& t = raw(r.keys[0]);
  switch (r.kind) {
    case Recipe::kConv3x3:
      pack_conv3x3_kernel<<<grid_for(r.numel), 256, 0, stream>>>(t.p(), r.out, static_cast<int>(t.shape[0]),
                                                                 static_cast<int>(t.shape[1]), r.cout_p, r.cin_p);
      break;
    case Recipe::kCatRows: {
      size_t off = 0;
      for (auto& k : r.keys) {
        const Weight& s = raw(k);
        CFGPP_CHECK_CUDA(cudaMemcpyAsync(r.out + off, s.p(), s.numel() * sizeof(__half), cudaMemcpyDeviceToDevice, stream));
        off += s.numel();
      }
      break;
    }
    case Recipe::kGeglu:
      pack_geglu_kernel<<<grid_for(r.numel), 256, 0, stream>>>(t.p(), r.out, static_cast<int>(t.shape[0]) / 2,
                                                               r.is_bias ? 1 : static_cast<int>(t.shape[1]));
      break;
    case Recipe::kHeadsRows: {
      HeadMats mats{};
      for (size_t i = 0; i < r.keys.size(); ++i) mats.p[i] = plain(r.keys[i]);
      const int K = static_cast<int>(r.numel / (r.keys.size() * r.heads * r.hdp));
      pack_heads_rows_kernel<<<grid_for(r.numel), 256, 0, stream>>>(mats, r.out, static_cast<int>(r.keys.size()),
                                                                    r.heads, r.hd, r.hdp, K);
      break;
    }
    case Recipe::kHeadsCols:
      pack_heads_cols_kernel<<<grid_for(r.numel), 256, 0, stream>>>(t.p(), r.out, static_cast<int>(t.shape[0]), r.heads,
                                                                    r.hd, r.hdp);
      break;
    case Recipe::kFoldLN:
      run_fold_ln(r.w_packed, plain(r.norm_prefix + ".weight"), plain(r.norm_prefix + ".bias"), r.bias_packed, r.fold.w,
                  r.fold.s, r.fold.t, r.N, r.K, stream);
      return 2 * r.numel * sizeof(__half) + 2 * static_cast<size_t>(r.N) * sizeof(float);
  }
  CFGPP_CHECK_CUDA(cudaGetLastError());
  return 2 * r.numel * sizeof(__half);
}

__half* WeightStore::packed_conv3x3(const std::string& key, int cin_p, int cout_p) {
  const Weight& t = raw(key);
  CFGPP_REQUIRE(t.shape.size() == 4 && t.shape[2] == 3 && t.shape[3] == 3, "expected (Cout,Cin,3,3): " + key);
  Recipe r{Recipe::kConv3x3, {key}};
  r.cin_p = cin_p ? cin_p : static_cast<int>(t.shape[1]);
  r.cout_p = cout_p ? cout_p : static_cast<int>(t.shape[0]);
  CFGPP_REQUIRE(r.cin_p >= t.shape[1] && r.cout_p >= t.shape[0], "padded conv narrower than its weight: " + key);
  r.numel = static_cast<size_t>(r.cout_p) * 9 * r.cin_p;
  return packed("conv3x3:" + key, r);
}

__half* WeightStore::packed_cat_rows(const std::vector<std::string>& keys) {
  Recipe r{Recipe::kCatRows, keys};
  for (auto& k : keys) r.numel += raw(k).numel();
  return packed(joined("cat", keys), r);
}

__half* WeightStore::packed_geglu(const std::string& key, bool is_bias) {
  const Weight& t = raw(key);
  CFGPP_REQUIRE(t.shape[0] % 256 == 0, "GEGLU width must be a multiple of 256: " + key);
  Recipe r{Recipe::kGeglu, {key}, t.numel()};
  r.is_bias = is_bias;
  return packed("geglu:" + key, r);
}

__half* WeightStore::packed_heads_rows(const std::vector<std::string>& keys, int heads, int hd, int hdp) {
  if (hd == hdp) return keys.size() == 1 ? plain(keys[0]) : packed_cat_rows(keys);
  CFGPP_REQUIRE(keys.size() <= 3, "at most three stacked projections");
  const size_t rows = static_cast<size_t>(heads) * hd;
  const size_t K = raw(keys[0]).numel() / rows;
  for (auto& k : keys) {
    const Weight& t = raw(k);
    CFGPP_REQUIRE(!t.shape.empty() && static_cast<size_t>(t.shape[0]) == rows && t.numel() == rows * K,
                  "unexpected projection shape: " + k);
  }
  Recipe r{Recipe::kHeadsRows, keys, keys.size() * heads * hdp * K};
  r.heads = heads;
  r.hd = hd;
  r.hdp = hdp;
  return packed(joined("heads_rows", keys), r);
}

__half* WeightStore::packed_heads_cols(const std::string& key, int heads, int hd, int hdp) {
  if (hd == hdp) return plain(key);
  const Weight& t = raw(key);
  CFGPP_REQUIRE(!t.shape.empty() && t.numel() == static_cast<size_t>(t.shape[0]) * heads * hd,
                "unexpected shape of a head-padded matrix: " + key);
  Recipe r{Recipe::kHeadsCols, {key}, static_cast<size_t>(t.shape[0]) * heads * hdp};
  r.heads = heads;
  r.hd = hd;
  r.hdp = hdp;
  return packed("heads_cols:" + key, r);
}

FoldedLN WeightStore::folded_ln(const std::string& name, const std::vector<std::string>& keys, const __half* w_packed,
                                int N, int K, const std::string& norm_prefix, const __half* bias_packed) {
  auto it = packed_.find("fold:" + name);
  if (it != packed_.end()) return it->second.fold;
  Recipe r{Recipe::kFoldLN, keys, static_cast<size_t>(N) * K};
  r.fold = {arena_.alloc<__half>(r.numel), arena_.alloc<float>(N), arena_.alloc<float>(N)};
  r.out = r.fold.w;
  r.w_packed = w_packed;
  r.bias_packed = bias_packed;
  r.norm_prefix = norm_prefix;
  r.N = N;
  r.K = K;
  run(r, nullptr);
  return packed_.emplace("fold:" + name, std::move(r)).first->second.fold;
}

size_t WeightStore::refresh(const std::set<std::string>& keys, cudaStream_t stream) {
  size_t bytes = 0;
  for (bool folds : {false, true})  // a fold reads the packed matrix: it runs after the packers
    for (auto& kv : packed_) {
      const Recipe& r = kv.second;
      if ((r.kind == Recipe::kFoldLN) == folds &&
          std::any_of(r.keys.begin(), r.keys.end(), [&](const std::string& k) { return keys.count(k) != 0; }))
        bytes += run(r, stream);
    }
  return bytes;
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
