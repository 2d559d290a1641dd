// cfgpp_b200 — LoRA merge: out[n,k] = fp16( fp32(base[n,k]) + sum_a c_a * sum_r up_a[n,r] * down_a[r,k] ).
// One 64 x 64 tile of the weight per CTA of 4 warps; every adapter's rank is walked in chunks of 32 through shared
// memory, the products run on mma.sync m16n8k16 with fp32 accumulators (two fp16 factors multiply exactly in fp32),
// each adapter's sum is scaled by its fp32 coefficient, and the tile is rounded to fp16 once. The job is bound by the
// base read and the merged write; tensor cores keep the rank-128 sum from costing as much as that traffic.
#include "executor.cuh"

namespace cfgpp {

namespace {

constexpr int TN = 64, TK = 64, RC = 32, THREADS = 128;

__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack2(__half lo, __half hi) {
  return static_cast<uint32_t>(__half_as_ushort(lo)) | (static_cast<uint32_t>(__half_as_ushort(hi)) << 16);
}

// rows x cols panel of src (leading dimension ld, origin (r0, c0), valid extent R x C) into shared memory with row
// stride LD, zero outside the valid extent. vec: 16-byte loads (ld % 8 == 0, C % 8 == 0, src 16-byte aligned).
template <int ROWS, int COLS, int LD>
__device__ __forceinline__ void load_panel(__half* dst, const __half* __restrict__ src, int ld, int r0, int c0, int R,
                                           int C, bool vec) {
  for (int i = threadIdx.x; i < ROWS * COLS / 8; i += THREADS) {
    const int row = i / (COLS / 8), col = (i % (COLS / 8)) * 8;
    const int r = r0 + row, c = c0 + col;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < R && c < C) {
      const __half* p = src + static_cast<size_t>(r) * ld + c;
      if (vec) {
        v = *reinterpret_cast<const uint4*>(p);
      } else {
        __half h[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = (c + j < C) ? p[j] : __ushort_as_half(0);
        v = make_uint4(pack2(h[0], h[1]), pack2(h[2], h[3]), pack2(h[4], h[5]), pack2(h[6], h[7]));
      }
    }
    *reinterpret_cast<uint4*>(dst + row * LD + col) = v;
  }
}

__global__ void __launch_bounds__(THREADS) lora_merge_kernel(const __half* __restrict__ base,
                                                             const __grid_constant__ LoraMergeArgs a, int N,
                                                             int K, __half* __restrict__ out, int vec_w) {
  __shared__ __align__(16) __half s_up[TN * (RC + 8)];
  __shared__ __align__(16) __half s_down[RC * (TK + 8)];
  __shared__ __align__(16) float s_delta[TN * (TK + 4)];
  const int n0 = blockIdx.y * TN, k0 = blockIdx.x * TK;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int g = lane / 4, q = lane % 4;

  float total[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) total[i][j] = 0.f;

  for (int ad = 0; ad < a.n; ++ad) {
    const int r = a.rank[ad];
    const bool vec_up = (r % 8 == 0) && (reinterpret_cast<uintptr_t>(a.up[ad]) % 16 == 0);
    const bool vec_down = (K % 8 == 0) && (reinterpret_cast<uintptr_t>(a.down[ad]) % 16 == 0);
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int rc = 0; rc < r; rc += RC) {
      __syncthreads();
      load_panel<TN, RC, RC + 8>(s_up, a.up[ad], r, n0, rc, N, r, vec_up);
      load_panel<RC, TK, TK + 8>(s_down, a.down[ad], K, rc, k0, r, K, vec_down);
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < RC; kk += 16) {
        if (rc + kk >= r) break;  // the rest of this chunk is zero padding
        const __half* ua = s_up + (warp * 16 + g) * (RC + 8) + kk + q * 2;
        uint32_t af[4];
        af[0] = *reinterpret_cast<const uint32_t*>(ua);
        af[1] = *reinterpret_cast<const uint32_t*>(ua + 8 * (RC + 8));
        af[2] = *reinterpret_cast<const uint32_t*>(ua + 8);
        af[3] = *reinterpret_cast<const uint32_t*>(ua + 8 * (RC + 8) + 8);
        const __half* db = s_down + (kk + q * 2) * (TK + 8) + g;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const __half* d = db + nt * 8;
          const uint32_t b0 = pack2(d[0], d[TK + 8]);
          const uint32_t b1 = pack2(d[8 * (TK + 8)], d[9 * (TK + 8)]);
          mma_16816(acc[nt], af, b0, b1);
        }
      }
    }
    const float c = a.coef[ad];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) total[i][j] = fmaf(c, acc[i][j], total[i][j]);
  }

  // stage the fp32 delta so that the base read and the merged write are 16 bytes per thread along k
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    float* d = s_delta + (warp * 16 + g) * (TK + 4) + nt * 8 + q * 2;
    *reinterpret_cast<float2*>(d) = make_float2(total[nt][0], total[nt][1]);
    *reinterpret_cast<float2*>(d + 8 * (TK + 4)) = make_float2(total[nt][2], total[nt][3]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < TN * TK / 8; i += THREADS) {
    const int row = i / (TK / 8), col = (i % (TK / 8)) * 8;
    const int n = n0 + row, k = k0 + col;
    if (n >= N || k >= K) continue;
    const float* d = s_delta + row * (TK + 4) + col;
    const size_t off = static_cast<size_t>(n) * K + k;
    if (vec_w) {
      const uint4 b = *reinterpret_cast<const uint4*>(base + off);
      const __half2* bh = reinterpret_cast<const __half2*>(&b);
      uint4 o;
      __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(bh[j]);
        oh[j] = __halves2half2(__float2half_rn(f.x + d[2 * j]), __float2half_rn(f.y + d[2 * j + 1]));
      }
      *reinterpret_cast<uint4*>(out + off) = o;
    } else {
      for (int j = 0; j < 8 && k + j < K; ++j) out[off + j] = __float2half_rn(__half2float(base[off + j]) + d[j]);
    }
  }
}

}  // namespace

void run_lora_merge(const __half* base, const LoraMergeArgs& a, int N, int K, __half* out, cudaStream_t stream) {
  CFGPP_REQUIRE(N >= 1 && K >= 1, "LoRA merge needs a non-empty [N, K] weight");
  CFGPP_REQUIRE(a.n >= 0 && a.n <= kMaxLoraPerTarget, "at most 4 adapters merge into one weight");
  for (int i = 0; i < a.n; ++i)
    CFGPP_REQUIRE(a.rank[i] >= 1 && a.rank[i] <= kMaxLoraRank && a.down[i] && a.up[i], "LoRA rank must be 1..128");
  const bool vec = (K % 8 == 0) && (reinterpret_cast<uintptr_t>(base) % 16 == 0) &&
                   (reinterpret_cast<uintptr_t>(out) % 16 == 0);
  const dim3 grid((K + TK - 1) / TK, (N + TN - 1) / TN);
  CFGPP_REQUIRE(grid.y <= 65535, "LoRA merge: too many rows");
  lora_merge_kernel<<<grid, THREADS, 0, stream>>>(base, a, N, K, out, vec ? 1 : 0);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

}  // namespace cfgpp
