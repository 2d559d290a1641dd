// cfgpp_b200 — what the UNet, VAE and CLIP executors share on the host side: the device memory they own, the weights
// they ingest by key (and the 3x3 convolution repack both image models need), and their stream-K workspace.
#pragma once
#include <map>
#include <memory>
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

// The raw fp16 weights of one model by key, plus the arena its repacked weights are allocated from.
class WeightStore {
 public:
  struct Weight {
    struct Free {
      void operator()(__half* p) const { cudaFree(p); }
    };
    std::unique_ptr<__half, Free> data;
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
  __half* packed_conv3x3(const std::string& key);                    // (Cout,Cin,3,3) -> [Cout][tap][Cin], cached
  template <typename T = __half>
  T* alloc(size_t n) {
    return packed_.alloc<T>(n);
  }

 private:
  std::map<std::string, Weight> raw_;
  std::map<std::string, __half*> conv3x3_;
  DeviceArena packed_;
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
