// cfgpp_b200 — host-side helpers: error handling, TMA tensor-map encoding (driver entry point fetched at
// run time so the library does not link libcuda), device properties.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>
#include <string>
#include <utility>

namespace cfgpp {

struct Error : public std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define CFGPP_CHECK_CUDA(expr)                                                                     \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      throw ::cfgpp::Error(-2, std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " at " + \
                                   __FILE__ + ":" + std::to_string(__LINE__));                     \
  } while (0)

#define CFGPP_REQUIRE(cond, msg)                                                                          \
  do {                                                                                                    \
    if (!(cond))                                                                                          \
      throw ::cfgpp::Error(-1, std::string("requirement failed: ") + #cond + " — " + (msg) + " at " +     \
                                   __FILE__ + ":" + std::to_string(__LINE__));                            \
  } while (0)

int num_sms();

// Launch with programmatic dependent launch enabled (see common.cuh). Capturable into CUDA graphs.
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                       Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  CFGPP_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...));
}

// Generic fp16 tiled tensor map, 128B swizzle. dims/strides innermost first; strides[i] is the byte
// stride of dim i+1 (dim 0 is contiguous). OOB elements are zero-filled by the hardware.
// `elem_strides` (optional, per dim): traversal stride — with stride s a box extent b loads ceil(b / s) elements
// (every s-th one from the box origin); used by the stride-2 convolution.
CUtensorMap make_tmap_f16(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box, int swizzle_bytes = 128, const uint32_t* elem_strides = nullptr);

// fp16 im2col tensor map (rank 3..5, dims / strides as above, NHWC-like: dim 0 = channels, last dim = images).
// A load walks `pixels_per_column` consecutive pixels of the bounding box in W, H, (D,) N order — wrapping at row and
// image ends — and fetches `channels_per_pixel` channels of each. Along each spatial dim the box spans coordinates
// [lower, dim - 1 + upper] (per-dim arrays, innermost spatial dim first; rank 4: each in [-128, 127]) and the walk
// takes every elem_strides[i]-th one from `lower`; the load's 16-bit offsets shift every pixel it reads (the filter
// tap), out-of-bounds pixels are zero-filled.
CUtensorMap make_tmap_im2col_f16(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                                 const int* lower, const int* upper, uint32_t channels_per_pixel,
                                 uint32_t pixels_per_column, const uint32_t* elem_strides, int swizzle_bytes = 128);

// 2D row-major [rows][cols] fp16 with leading dimension ld (elements); box = (64 cols, box_rows).
CUtensorMap make_tmap_2d(const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);
// epilogue tiles: box = (32 cols = 64 B, box_rows), 64B swizzle (output stores / residual loads)
CUtensorMap make_tmap_2d_sw64(const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);

}  // namespace cfgpp
