// cfgpp_b200 — what the UNet, VAE and CLIP executors share on the host side: the device memory they own, the weights
// they ingest by key and every repack of them a kernel reads, and their stream-K workspace.
#pragma once
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "host.h"

namespace cfgpp {

// Grid of a grid-stride kernel with 256-thread blocks over n elements.
int grid_for(size_t n);

// Device allocations owned, counted and freed together. Every allocation is rounded up to a multiple of 256 B (at
// least 256 B); bytes() is the sum of the rounded requests.
class DeviceArena {
 public:
  DeviceArena() = default;
  ~DeviceArena() { clear(); }
  DeviceArena(const DeviceArena&) = delete;
  DeviceArena& operator=(const DeviceArena&) = delete;

  void* alloc(size_t bytes);
  template <typename T>
  T* alloc(size_t n) {
    return static_cast<T*>(alloc(n * sizeof(T)));
  }
  size_t bytes() const { return bytes_; }
  void clear();

 private:
  std::vector<void*> ptrs_;
  size_t bytes_ = 0;
};

// ---- lora.cu ---------------------------------------------------------------------------------------------------
constexpr int kMaxLoraPerTarget = 4;
constexpr int kMaxLoraRank = 128;
// The adapters merged into one weight: down_a [rank_a][K], up_a [N][rank_a] fp16 (device), coef_a fp32.
struct LoraMergeArgs {
  const __half* down[kMaxLoraPerTarget];
  const __half* up[kMaxLoraPerTarget];
  int rank[kMaxLoraPerTarget];
  float coef[kMaxLoraPerTarget];
  int n;
};
// out[n,k] = fp16(fp32(base[n,k]) + sum_a coef_a * sum_r up_a[n,r] * down_a[r,k]): fp32 accumulation on the tensor
// cores, one rounding. Any N, K; ranks 1..128. out may be base.
void run_lora_merge(const __half* base, const LoraMergeArgs& a, int N, int K, __half* out, cudaStream_t stream);

// A weight [N][K] with a LayerNorm folded in (run_fold_ln): w = fp16(w * gamma), s and t [N] fp32.
struct FoldedLN {
  __half* w;
  float* s;
  float* t;
};

// The raw fp16 weights of one model by key, and every packed operand derived from them. Each packed buffer remembers
// its recipe, so that refresh can derive it again in place when the raw weights change.
class WeightStore {
 public:
  struct Weight {
    struct Free {
      void operator()(__half* p) const { cudaFree(p); }
    };
    using Ptr = std::unique_ptr<__half, Free>;
    Ptr data;
    std::vector<int64_t> shape;
    __half* p() const { return data.get(); }
    size_t numel() const;
  };

  // fp16 is copied, fp32 converted to fp16 (on `stream`); a key loaded again replaces the earlier tensor
  void load(const std::string& key, const void* data, const int64_t* shape, int ndim, int dtype, cudaStream_t stream);
  bool has(const std::string& key) const { return raw_.count(key) != 0; }
  const Weight& raw(const std::string& key) const;  // Error -10 "missing weight: <key>"
  __half* plain(const std::string& key) const { return raw(key).p(); }
  __half* plain(const std::string& key, size_t expect_numel) const;  // Error -11 on a size mismatch

  // ---- packed operands, cached by name. The first call packs on the legacy stream, so the caller synchronises the
  // stream the weights were loaded on first; later calls return the same pointer ----
  // (Cout,Cin,3,3) -> [cout_p][tap][cin_p], zero beyond Cout / Cin (0: unpadded)
  __half* packed_conv3x3(const std::string& key, int cin_p = 0, int cout_p = 0);
  __half* packed_cat_rows(const std::vector<std::string>& keys);  // the tensors one after the other
  // GEGLU proj (2*inner, K) or its bias (2*inner): per 128 rows, value / gate halves interleaved into 256-row tiles
  __half* packed_geglu(const std::string& key, bool is_bias);
  // Every source viewed as [shape[0]][numel / shape[0]] (a bias is a K = 1 matrix), each head's hd rows / columns
  // zero-padded to hdp: rows stacks up to three (heads*hd, K) sources into [(source, head, hdp)][K], cols turns
  // (N, heads*hd) into (N, heads*hdp). heads = 1 is a plain row / column pad; hd == hdp returns the raw tensor or the
  // row concatenation.
  __half* packed_heads_rows(const std::vector<std::string>& keys, int heads, int hd, int hdp);
  __half* packed_heads_cols(const std::string& key, int heads, int hd, int hdp);
  // the LayerNorm `norm_prefix` folded into w_packed [N][K] and bias_packed [N] (may be null), which were packed from
  // `keys`
  FoldedLN folded_ln(const std::string& name, const std::vector<std::string>& keys, const __half* w_packed, int N, int K,
                     const std::string& norm_prefix, const __half* bias_packed);
  // derives again, on `stream`, every packed operand that reads one of `keys` (folds after the packers); returns the
  // bytes read + written
  size_t refresh(const std::set<std::string>& keys, cudaStream_t stream);

  // ---- LoRA adapters: W_eff = fp16(fp32(W) + sum_a c_a up_a down_a), c_a = scale_a * alpha_a / rank_a, always merged
  // from a pristine copy of W into the raw tensor's own storage (pointers handed out by plain() stay valid) ----
  // Adds adapter `adapter`'s factors for `key`: down [rank][K], up [N][rank] (device, fp16 or fp32 rounded to fp16),
  // N = shape[0] and K = numel / N of raw(key). The key's first adapter takes its pristine backup. Nothing is merged
  // until lora_apply.
  void lora_add(int adapter, const std::string& key, const void* down, const void* up, int rank, float alpha, int dtype,
                cudaStream_t stream);
  // Merges every target at `scales` (one per adapter id 0..n-1) on `stream`; returns the keys written and adds the
  // bytes read + written to *bytes.
  std::set<std::string> lora_apply(const float* scales, int n, cudaStream_t stream, size_t* bytes);
  // Copies every backup over its raw tensor on `stream` (the base bits) and returns those keys; lora_free then
  // synchronises `stream` and releases factors and backups.
  std::set<std::string> lora_restore(cudaStream_t stream, size_t* bytes);
  void lora_free(cudaStream_t stream);
  int lora_adapters() const { return lora_adapters_; }
  int lora_targets() const { return static_cast<int>(lora_.size()); }
  size_t lora_backup_bytes() const;

 private:
  // How one packed buffer is derived from raw weights, so that it can be derived again into the same buffer.
  struct Recipe {
    enum Kind { kConv3x3, kCatRows, kGeglu, kHeadsRows, kHeadsCols, kFoldLN } kind;
    std::vector<std::string> keys;  // the raw weights it reads
    size_t numel = 0;               // of out
    __half* out = nullptr;
    int cin_p = 0, cout_p = 0;       // kConv3x3
    bool is_bias = false;            // kGeglu
    int heads = 0, hd = 0, hdp = 0;  // kHeadsRows, kHeadsCols
    // kFoldLN: the LayerNorm `norm_prefix` folded into the packed w [N][K] and bias; out is fold.w
    FoldedLN fold{};
    const __half *w_packed = nullptr, *bias_packed = nullptr;
    std::string norm_prefix;
    int N = 0, K = 0;
  };
  __half* packed(const std::string& name, Recipe r);  // returns the cached buffer, or allocates and packs it
  size_t run(const Recipe& r, cudaStream_t stream);   // returns bytes read + written

  struct LoraFactor {
    int adapter, rank;
    float alpha;
    Weight::Ptr down, up;
  };
  struct LoraTarget {
    Weight::Ptr backup;
    std::vector<LoraFactor> factors;
  };
  std::map<std::string, Weight> raw_;
  std::map<std::string, Recipe> packed_;
  std::map<std::string, LoraTarget> lora_;
  int lora_adapters_ = 0;  // highest adapter id added + 1
  DeviceArena arena_;  // the packed buffers
};

// One handle's stream-K buffer pair on `device`; plan building selects it with a StreamKScope (gemm.cuh).
class StreamKWorkspace {
 public:
  explicit StreamKWorkspace(int device);
  ~StreamKWorkspace();
  StreamKWorkspace(const StreamKWorkspace&) = delete;
  StreamKWorkspace& operator=(const StreamKWorkspace&) = delete;
  float* ws() const { return ws_; }
  unsigned* flags() const { return flags_; }

 private:
  float* ws_ = nullptr;
  unsigned* flags_ = nullptr;
};

}  // namespace cfgpp
