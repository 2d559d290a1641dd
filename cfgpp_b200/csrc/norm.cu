// cfgpp_b200 — GroupNorm(32)(+SiLU) and LayerNorm on NHWC / token-major fp16 activations (HBM-bound kernels).
//
// Numerics follow the reference's autocast graph: statistics and the affine transform (and SiLU) are computed
// in fp32 from the fp16 input, and the result is rounded to fp16 exactly once — the point where the reference's
// fp32 norm output is cast for the following conv / linear.
//
// GroupNorm is two launches: (1) per-(sample, pixel-chunk) partial (mean, M2) per group — deterministic, no atomics in
// global memory; (2) apply, which merges the partials on the fly. Both take an optional second source so that
// torch.cat([h, skip], dim=1) of the up-blocks is never materialised un-normalised.
//
// The LayerNorm fold of the transformer blocks (see GemmParams in gemm.cuh) prepares its weights here too.
#include "common.cuh"
#include "ops.cuh"

namespace cfgpp {

namespace {

constexpr int GROUPS = 32;

struct GnSrc {
  const __half* x1;
  const __half* x2;
  int C1, C2;
};

CFGPP_DEVICE uint4 load_vec(const GnSrc& s, size_t pix, int c) {  // c multiple of 8, never straddles C1
  if (c < s.C1) return *reinterpret_cast<const uint4*>(s.x1 + pix * s.C1 + c);
  return *reinterpret_cast<const uint4*>(s.x2 + pix * s.C2 + (c - s.C1));
}

// Chan et al.'s pairwise update: a set of na elements absorbs a disjoint set (nb > 0, mean_b, m2_b), m2 being the sum of
// squared deviations from the set's mean. Every term of the new m2 is >= 0, so nothing cancels. The running mean is
// kept as ref + off, ref the first set's mean: a chain of merges then rounds at the scale of the spread between the
// sets' means, not at that of the mean itself (a mean far from 0 would cost one rounding of it per merge).
CFGPP_DEVICE void chan_merge(float& ref, float& off, float& m2, float na, float nb, float mean_b, float m2_b) {
  if (na == 0.f) {
    ref = mean_b;
    off = 0.f;
    m2 = m2_b;
    return;
  }
  const float f = __fdividef(nb, na + nb);  // a weight: its 2-ulp error scales d, never the mean itself
  const float d = (mean_b - ref) - off;
  off += d * f;
  m2 += m2_b + d * d * (na * f);
}

// pixels of chunk i, and of the chunks i, i + 8, ... whose partials one of the apply's 8 reduction parts merges
CFGPP_DEVICE int gn_chunk_pixels(int i, int ppb, int HW) { return min(ppb, HW - i * ppb); }
CFGPP_DEVICE int gn_part_pixels(int part, int nchunk, int ppb, int HW) {
  int n = 0;
  for (int i = part; i < nchunk; i += 8) n += gn_chunk_pixels(i, ppb, HW);
  return n;
}

// grid (nchunk, B); block = vpp * k threads (vpp = C / 8 vectors per pixel) so a thread keeps one channel vector and
// walks every pstep-th pixel of the chunk (up to 2048 of them at the VAE's 1024^2 levels).
//
// A thread's statistics come in runs of up to kRunPx pixels: fp32 sums of x - K and (x - K)^2, K the run's own first
// value, so the shifted sums only cancel over the run's own spread (an outlier of the group costs at most the run it
// shifts). A finished run becomes (mean, M2) and is merged into the thread's summary by chan_merge; the threads'
// slots are then merged per group in a fixed order. Counts are never stored: every level recomputes them from the
// launch geometry. At most 768 threads (C <= 6144, see run_groupnorm), so at most 80 registers a thread.
__global__ void __launch_bounds__(768)
    gn_stats_kernel(GnSrc src, int HW, int C, int px_per_block, float* __restrict__ partial) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float sm[];  // [pstep][C] means, then [pstep][C] M2s (one slot per thread: no atomics)
  const int vpp = C >> 3;
  const int cpg = C / GROUPS;
  const int b = blockIdx.y;
  const int chunk = blockIdx.x;
  const int vec = threadIdx.x % vpp;
  const int prow = threadIdx.x / vpp;
  const int pstep = blockDim.x / vpp;
  float s[8], q[8], piv[8], ref[8], off[8], m2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = q[i] = piv[i] = ref[i] = off[i] = m2[i] = 0.f;
  int nrun = 0, nthr = 0;  // pixels of the open run; pixels already merged into (ref + off, m2)
  auto set_pivot = [&](const uint4& u) {
    const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
    for (int i = 0; i < 8; ++i) piv[i] = __half2float(h[i]);
  };
  // x - K is exact when x and K are within a factor of 2 (Sterbenz); otherwise it rounds once, like any fp32 sum term
  auto accumulate = [&](const uint4& u) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      const float d0 = f.x - piv[2 * i], d1 = f.y - piv[2 * i + 1];
      s[2 * i] += d0;
      q[2 * i] += d0 * d0;
      s[2 * i + 1] += d1;
      q[2 * i + 1] += d1 * d1;
    }
  };
  auto fold = [&]() {
    if (nrun == 0) return;
    const float nr = static_cast<float>(nrun), rn = __frcp_rn(nr);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float dm = s[i] * rn;
      chan_merge(ref[i], off[i], m2[i], static_cast<float>(nthr), nr, piv[i] + dm, fmaxf(q[i] - s[i] * dm, 0.f));
      s[i] = q[i] = 0.f;
    }
    nthr += nrun;
    nrun = 0;
  };
  const int p0 = chunk * px_per_block;
  const int pend = min(px_per_block, HW - p0);
  const size_t base = static_cast<size_t>(b) * HW + p0;
  constexpr int U = 4;        // independent 16 B loads in flight per thread
  constexpr int kRunPx = 32;  // pixels per run (a multiple of U; the tail loop below adds at most U - 1)
  int pp = prow;
  for (; pp + (U - 1) * pstep < pend; pp += U * pstep) {
    uint4 u[U];
#pragma unroll
    for (int j = 0; j < U; ++j) u[j] = load_vec(src, base + pp + j * pstep, vec * 8);
    if (nrun == 0) set_pivot(u[0]);
#pragma unroll
    for (int j = 0; j < U; ++j) accumulate(u[j]);
    nrun += U;
    if (nrun == kRunPx) fold();
  }
  for (; pp < pend; pp += pstep) {
    const uint4 u = load_vec(src, base + pp, vec * 8);
    if (nrun == 0) set_pivot(u);
    accumulate(u);
    ++nrun;
  }
  fold();
  float* sq = sm + pstep * C;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sm[prow * C + vec * 8 + i] = ref[i] + off[i];
    sq[prow * C + vec * 8 + i] = m2[i];
  }
  __syncthreads();
  if (threadIdx.x < GROUPS) {  // fixed merge order -> bit-reproducible statistics
    float a = 0.f, o = 0.f, m = 0.f, n = 0.f;
    for (int r = 0; r < pstep && r < pend; ++r) {
      const float nr = static_cast<float>((pend - 1 - r) / pstep + 1);  // pixels of the threads in row r
      for (int i = 0; i < cpg; ++i) {
        chan_merge(a, o, m, n, nr, sm[r * C + threadIdx.x * cpg + i], sq[r * C + threadIdx.x * cpg + i]);
        n += nr;
      }
    }
    float* dst = partial + ((static_cast<size_t>(b) * gridDim.x + chunk) * GROUPS + threadIdx.x) * 2;
    dst[0] = a + o;
    dst[1] = m;
  }
}

// grid (nchunk, B); block = vpp * k threads: a thread owns one 8-channel vector, so the per-channel affine
// (x - mean) * a + beta (a = rstd * gamma) uses 24 registers set up once per thread.
__global__ void gn_apply_kernel(GnSrc src, int HW, int C, int px_per_block, const float* __restrict__ partial,
                                int nchunk, const __half* __restrict__ gamma, const __half* __restrict__ beta,
                                float eps, int silu, __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_mean[GROUPS], s_rstd[GROUPS];
  __shared__ float2 s_part[8][GROUPS];
  const int b = blockIdx.y;
  const int cpg = C / GROUPS;
  // Cross-chunk merge of the partials, spread over 8 x 32 threads (each merges every 8th chunk, loads independent),
  // then combined in a fixed order: a single thread per group walking all (up to 128) chunks exposed ~10 us of
  // serialised L2 latency at the head of EVERY block.
  for (int idx = threadIdx.x; idx < 8 * GROUPS; idx += blockDim.x) {
    const int g = idx & (GROUPS - 1), part = idx / GROUPS;
    float a = 0.f, o = 0.f, m = 0.f, n = 0.f;
    const float* src_p = partial + (static_cast<size_t>(b) * nchunk * GROUPS + g) * 2;
    for (int i = part; i < nchunk; i += 8) {
      const float2 v = *reinterpret_cast<const float2*>(src_p + static_cast<size_t>(i) * GROUPS * 2);
      const float ni = static_cast<float>(gn_chunk_pixels(i, px_per_block, HW) * cpg);
      chan_merge(a, o, m, n, ni, v.x, v.y);
      n += ni;
    }
    s_part[part][g] = make_float2(a + o, m);
  }
  __syncthreads();
  if (threadIdx.x < GROUPS) {
    float a = 0.f, o = 0.f, m = 0.f, n = 0.f;
    for (int part = 0; part < 8 && part < nchunk; ++part) {
      const float np = static_cast<float>(gn_part_pixels(part, nchunk, px_per_block, HW) * cpg);
      chan_merge(a, o, m, n, np, s_part[part][threadIdx.x].x, s_part[part][threadIdx.x].y);
      n += np;
    }
    s_mean[threadIdx.x] = a + o;
    s_rstd[threadIdx.x] = rsqrtf(m / (static_cast<float>(HW) * (C / GROUPS)) + eps);
  }
  __syncthreads();
  const int vpp = C >> 3;
  const int vec = threadIdx.x % vpp;
  const int prow = threadIdx.x / vpp;
  const int pstep = blockDim.x / vpp;
  const int c0 = vec * 8;
  const uint4 ug = *reinterpret_cast<const uint4*>(gamma + c0);
  const uint4 ub = *reinterpret_cast<const uint4*>(beta + c0);
  const __half* hg = reinterpret_cast<const __half*>(&ug);
  const __half* hb = reinterpret_cast<const __half*>(&ub);
  float mu[8], sc[8], sh[8];  // mean, a, beta of each of this thread's 8 channels
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int g = (c0 + k) / cpg;
    mu[k] = s_mean[g];
    sc[k] = s_rstd[g] * __half2float(hg[k]);
    sh[k] = __half2float(hb[k]);
  }
  const int p0 = blockIdx.x * px_per_block;
  const int pend = min(px_per_block, HW - p0);
  const size_t base = static_cast<size_t>(b) * HW + p0;
  constexpr int U = 4;
  auto emit = [&](const uint4& u, size_t gp) {
    const __half* hx = reinterpret_cast<const __half*>(&u);
    float y[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float v = (__half2float(hx[k]) - mu[k]) * sc[k] + sh[k];
      if (silu) v = silu_f(v);
      y[k] = v;
    }
    uint4 o;
    o.x = pack_half2(y[0], y[1]);
    o.y = pack_half2(y[2], y[3]);
    o.z = pack_half2(y[4], y[5]);
    o.w = pack_half2(y[6], y[7]);
    *reinterpret_cast<uint4*>(out + gp * C + c0) = o;
  };
  int pp = prow;
  for (; pp + (U - 1) * pstep < pend; pp += U * pstep) {
    uint4 u[U];
#pragma unroll
    for (int j = 0; j < U; ++j) u[j] = load_vec(src, base + pp + j * pstep, c0);
#pragma unroll
    for (int j = 0; j < U; ++j) emit(u[j], base + pp + j * pstep);
  }
  for (; pp < pend; pp += pstep) emit(load_vec(src, base + pp, c0), base + pp);
}

// LayerNorm of one row xr [C] by one warp (C % 8 == 0, C <= 2048): fp32 statistics and affine transform, one fp16
// rounding; store(vi, o) writes the 8 outputs of columns [8 vi, 8 vi + 8). Every LayerNorm kernel runs this body, so a
// row normalised by any of them has the same bits.
template <typename Store>
CFGPP_DEVICE void layernorm_row(const __half* __restrict__ xr, int C, const __half* __restrict__ gamma,
                                const __half* __restrict__ beta, float eps, int lane, Store store) {
  const int nvec = C >> 3;
  constexpr int MAXV = 8;
  uint4 v[MAXV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      v[i] = *reinterpret_cast<const uint4*>(xr + vi * 8);
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __half22float2(h[k]);
        sum += f.x + f.y;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __half22float2(h[k]);
        sq += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const uint4 ug = *reinterpret_cast<const uint4*>(gamma + vi * 8);
      const uint4 ub = *reinterpret_cast<const uint4*>(beta + vi * 8);
      const __half* hx = reinterpret_cast<const __half*>(&v[i]);
      const __half* hg = reinterpret_cast<const __half*>(&ug);
      const __half* hb = reinterpret_cast<const __half*>(&ub);
      float y[8];
#pragma unroll
      for (int k = 0; k < 8; ++k)
        y[k] = (__half2float(hx[k]) - mean) * rstd * __half2float(hg[k]) + __half2float(hb[k]);
      uint4 o;
      o.x = pack_half2(y[0], y[1]);
      o.y = pack_half2(y[2], y[3]);
      o.z = pack_half2(y[4], y[5]);
      o.w = pack_half2(y[6], y[7]);
      store(vi, o);
    }
  }
}

// one warp per row; C % 8 == 0, C <= 2048
__global__ void layernorm_kernel(const __half* __restrict__ x, int M, int C, const __half* __restrict__ gamma,
                                 const __half* __restrict__ beta, float eps, __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  __half* orow = out + static_cast<size_t>(row) * C;
  layernorm_row(x + static_cast<size_t>(row) * C, C, gamma, beta, eps, lane,
                [=](int vi, const uint4& o) { *reinterpret_cast<uint4*>(orow + vi * 8) = o; });
}

// The two LayerNorms of a Resampler layer in one launch, one warp per row of kv [NB][T + Q][C]: row (b, j < T) is
// LN0(x[b, j]), row (b, T + i) is LN1(lat[b, i]), which also goes to q [NB][Q][C] (the query operand).
__global__ void ln_concat_kernel(const __half* __restrict__ x, const __half* __restrict__ lat, int NB, int T, int Q,
                                 int C, const __half* __restrict__ g0, const __half* __restrict__ b0,
                                 const __half* __restrict__ g1, const __half* __restrict__ b1, float eps,
                                 __half* __restrict__ kv, __half* __restrict__ q) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int S = T + Q;
  if (row >= NB * S) return;
  const int b = row / S, j = row - b * S;
  __half* kvrow = kv + static_cast<size_t>(row) * C;
  if (j < T) {
    layernorm_row(x + (static_cast<size_t>(b) * T + j) * C, C, g0, b0, eps, lane,
                  [=](int vi, const uint4& o) { *reinterpret_cast<uint4*>(kvrow + vi * 8) = o; });
  } else {
    const size_t r = static_cast<size_t>(b) * Q + (j - T);
    __half* qrow = q + r * C;
    layernorm_row(lat + r * C, C, g1, b1, eps, lane, [=](int vi, const uint4& o) {
      *reinterpret_cast<uint4*>(kvrow + vi * 8) = o;
      *reinterpret_cast<uint4*>(qrow + vi * 8) = o;
    });
  }
}

// LayerNorm fold (see GemmParams): one warp per (packed) weight row n
__global__ void fold_ln_kernel(const __half* __restrict__ w, const __half* __restrict__ gamma,
                               const __half* __restrict__ beta, const __half* __restrict__ bias,
                               __half* __restrict__ wf, float* __restrict__ s_out, float* __restrict__ t_out, int N,
                               int K) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float s = 0.f, t = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float wv = __half2float(w[static_cast<size_t>(n) * K + k]);
    const __half wg = __float2half_rn(wv * __half2float(gamma[k]));
    wf[static_cast<size_t>(n) * K + k] = wg;
    s += __half2float(wg);
    t += __half2float(beta[k]) * wv;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  if (lane == 0) {
    s_out[n] = s;
    t_out[n] = t + (bias ? __half2float(bias[n]) : 0.f);
  }
}

}  // namespace

// up to 128 pixel chunks per sample (the partial-sum buffer holds 128) so that even the 32x32 level launches
// >= 512 blocks; at least 4 pixels per block
int gn_px_per_block(int HW) {
  int ppb = (HW + 127) / 128;
  return ppb < 4 ? 4 : ppb;
}
int gn_num_chunks(int HW) { return (HW + gn_px_per_block(HW) - 1) / gn_px_per_block(HW); }
size_t gn_partial_floats(int B, int HW) { return static_cast<size_t>(B) * gn_num_chunks(HW) * GROUPS * 2; }

void run_groupnorm(const __half* x1, int C1, const __half* x2, int C2, int B, int HW, const __half* gamma,
                   const __half* beta, float eps, bool silu, float* partial, __half* out, cudaStream_t stream) {
  const int C = C1 + C2;
  CFGPP_REQUIRE(C % GROUPS == 0 && C % 8 == 0 && C1 % 8 == 0, "GroupNorm needs C % 32 == 0 and 8-aligned sources");
  GnSrc src{x1, x2 ? x2 : x1, C1, C2};
  const int vpp = C / 8;
  const int ppb = gn_px_per_block(HW);
  const int nchunk = gn_num_chunks(HW);
  int k = 256 / vpp;
  if (k < 1) k = 1;
  const int threads = vpp * k;
  const size_t stats_smem = 2 * static_cast<size_t>(k) * C * sizeof(float);
  // gn_stats_kernel keeps one (mean, M2) slot per thread and channel in the default 48 KB of dynamic shared memory
  // (no opt-in): C <= 6144, far above any model's channel count
  CFGPP_REQUIRE(threads <= 1024 && stats_smem <= 48 * 1024, "GroupNorm channel count too large (C <= 6144)");
  launch_pdl(gn_stats_kernel, dim3(nchunk, B), dim3(threads), stats_smem, stream, src, HW, C,
             ppb, partial);
  launch_pdl(gn_apply_kernel, dim3(nchunk, B), dim3(threads), 0, stream, src, HW, C, ppb, partial, nchunk, gamma, beta, eps,
                                                           silu ? 1 : 0, out);
}

void run_layernorm(const __half* x, int M, int C, const __half* gamma, const __half* beta, float eps, __half* out,
                   cudaStream_t stream) {
  CFGPP_REQUIRE(C % 8 == 0 && C <= 2048, "LayerNorm needs C % 8 == 0 and C <= 2048");
  const int warps = 8;
  launch_pdl(layernorm_kernel, dim3((M + warps - 1) / warps), dim3(warps * 32), 0, stream, x, M, C, gamma, beta, eps, out);
}

void run_ln_concat(const __half* x, const __half* lat, int NB, int T, int Q, int C, const __half* g0, const __half* b0,
                   const __half* g1, const __half* b1, float eps, __half* kv, __half* q, cudaStream_t stream) {
  CFGPP_REQUIRE(C % 8 == 0 && C <= 2048, "LayerNorm needs C % 8 == 0 and C <= 2048");
  CFGPP_REQUIRE(NB >= 1 && T >= 1 && Q >= 1, "empty LayerNorm concatenation");
  const int warps = 8, rows = NB * (T + Q);
  launch_pdl(ln_concat_kernel, dim3((rows + warps - 1) / warps), dim3(warps * 32), 0, stream, x, lat, NB, T, Q, C, g0, b0,
             g1, b1, eps, kv, q);
}

void run_fold_ln(const __half* w, const __half* gamma, const __half* beta, const __half* bias, __half* wf, float* s,
                 float* t, int N, int K, cudaStream_t stream) {
  const int warps = 8;
  fold_ln_kernel<<<(N + warps - 1) / warps, warps * 32, 0, stream>>>(w, gamma, beta, bias, wf, s, t, N, K);
  CFGPP_CHECK_CUDA(cudaGetLastError());
}

}  // namespace cfgpp
