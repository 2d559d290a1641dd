// cfgpp_b200 — host helpers (see host.h)
#include "host.h"

#include <cudaTypedefs.h>

#include <mutex>

namespace cfgpp {

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    CFGPP_CHECK_CUDA(cudaGetDevice(&dev));
    CFGPP_CHECK_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  }
  return n;
}

static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  if (!fn) throw Error(-3, "cuTensorMapEncodeTiled driver entry point unavailable (no CUDA driver?)");
  return fn;
}

CUtensorMap make_tmap_f16(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box, int swizzle_bytes, const uint32_t* elem_strides) {
  CUtensorMap m;
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = elem_strides ? elem_strides[i] : 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CFGPP_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16B aligned");
  for (int i = 0; i + 1 < rank; ++i) CFGPP_REQUIRE(gstr[i] % 16 == 0, "TMA strides must be multiples of 16B");
  CFGPP_REQUIRE(static_cast<int>(box[0]) * 2 <= swizzle_bytes, "inner box must fit the swizzle span");
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                              : swizzle_bytes == 64  ? CU_TENSOR_MAP_SWIZZLE_64B
                                                     : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstr, bx,
                               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Error(-4, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
  return m;
}

static PFN_cuTensorMapEncodeIm2col_v12000 get_encode_im2col_fn() {
  static PFN_cuTensorMapEncodeIm2col_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_cuTensorMapEncodeIm2col_v12000>(p);
  });
  if (!fn) throw Error(-3, "cuTensorMapEncodeIm2col driver entry point unavailable (no CUDA driver?)");
  return fn;
}

CUtensorMap make_tmap_im2col_f16(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                                 const int* lower, const int* upper, uint32_t channels_per_pixel,
                                 uint32_t pixels_per_column, const uint32_t* elem_strides, int swizzle_bytes) {
  CFGPP_REQUIRE(rank >= 3 && rank <= 5, "im2col tensor maps have rank 3..5");
  CUtensorMap m;
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t estr[5];
  const int lim = rank == 3 ? 32768 : (rank == 4 ? 128 : 16);  // corner offset range [-lim, lim - 1]
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    estr[i] = elem_strides ? elem_strides[i] : 1;
  }
  for (int i = 0; i + 2 < rank; ++i)
    CFGPP_REQUIRE(lower[i] >= -lim && lower[i] < lim && upper[i] >= -lim && upper[i] < lim,
                  "im2col pixel-box corner out of range for this rank");
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CFGPP_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16B aligned");
  for (int i = 0; i + 1 < rank; ++i) CFGPP_REQUIRE(gstr[i] % 16 == 0, "TMA strides must be multiples of 16B");
  CFGPP_REQUIRE(static_cast<int>(channels_per_pixel) * 2 <= swizzle_bytes, "pixel must fit the swizzle span");
  CFGPP_REQUIRE(pixels_per_column >= 1 && pixels_per_column <= 1024, "im2col pixels per column must be 1..1024");
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                              : swizzle_bytes == 64  ? CU_TENSOR_MAP_SWIZZLE_64B
                                                     : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = get_encode_im2col_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstr,
                                      lower, upper, channels_per_pixel, pixels_per_column, estr,
                                      CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Error(-4, "cuTensorMapEncodeIm2col failed with CUresult " + std::to_string((int)r));
  return m;
}

CUtensorMap make_tmap_2d(const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld * 2};
  uint32_t box[2] = {64, box_rows};
  return make_tmap_f16(base, 2, dims, strides, box);
}

CUtensorMap make_tmap_2d_sw64(const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld * 2};
  uint32_t box[2] = {32, box_rows};
  return make_tmap_f16(base, 2, dims, strides, box, 64);
}

}  // namespace cfgpp
