// cfgpp_b200 — flash-style attention forward on sm_90a tensor cores. See attention.cuh.
// Padded head dim 64 runs on the warp-specialised wgmma kernel attn64_kernel further down; head dims 128 and 192 on
// attn_kernel<HD> (mma.sync m16n8k16):
//
// One CTA = one 64-row query tile of one (batch, head), 4 warps of 16 query rows each, looping over 64-row KV tiles:
//   thread 0 : TMA producer (Q once; K / V into a 2-deep ring, 128B swizzle, mbarrier complete_tx)
//   all      : S = Q K^T (ldmatrix from the swizzled tiles, fp32 accumulators in registers), online softmax on the
//              accumulator fragments (running max and sum per row, exp2 with the scale folded in), P rounded to fp16
//              and fed straight back from registers as the A operand of O += P V (V through ldmatrix.trans).
// The same kernel serves self-attention (Nkv = Nq) and cross-attention (Nkv = 77 text tokens): a KV tile past Nkv is
// zero-filled by the TMA and its columns are masked to -inf. Head dims of 40 / 80 / 160 arrive zero-padded to 64 / 128
// / 192 columns; the padding columns of V are zero, so those of the output are too.
#include <cmath>
#include <type_traits>

#include "attention.cuh"
#include "common.cuh"

namespace cfgpp {

void attn_configure();

namespace {

constexpr int BQ = 64;
constexpr int BKV = 64;
constexpr int kThreads = 128;
constexpr int ATOM_BYTES = 64 * 64 * 2;  // 8 KB: one [64 rows x 64 fp16] swizzle-128B atom

template <int HD>
struct ACfg {
  static constexpr int NA = HD / 64;                  // swizzle atoms per tile row
  static constexpr int TILE_BYTES = NA * ATOM_BYTES;  // one Q / K / V tile
  static constexpr int SMEM_BYTES = TILE_BYTES * 5 + 1024 + 64;  // Q + 2 x K + 2 x V, alignment slack, barriers
  static_assert(SMEM_BYTES <= 232448, "shared memory overflow");
};

// byte offset of (row, 16-byte chunk) in a tile of NA atoms [64 rows x 128 B] (128B swizzle: chunk ^= row % 8)
CFGPP_DEVICE uint32_t tile_off(int row, int chunk) {
  return (chunk >> 3) * ATOM_BYTES + row * 128 + (((chunk & 7) ^ (row & 7)) << 4);
}

// IP: the decoupled cross-attention of attn_ip_kernel. After the text tiles, one more ring fill brings the image
// tokens' K / V (a 64-row tile of which the first p.Nkv2 rows are valid); their softmax has its own max and sum, and
// the output is O1 / l1 + s * O2 / l2 rounded once. s = 0 skips the image tile: the plain kernel's arithmetic exactly.
template <int HD, bool IP>
CFGPP_DEVICE void attn_body(const AttnParams& p, const CUtensorMap* map_q, const CUtensorMap* map_k,
                            const CUtensorMap* map_v, const CUtensorMap* map_k2, const CUtensorMap* map_v2) {
  using A = ACfg<HD>;
  constexpr int NA = A::NA;
  constexpr int TILE_BYTES = A::TILE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + TILE_BYTES;      // 2 tiles
  uint8_t* sV = sK + 2 * TILE_BYTES;  // 2 tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * TILE_BYTES);
  uint64_t* q_full = bars;        // [1]
  uint64_t* kv_full = bars + 1;   // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int head = blockIdx.y;
  const int batch = blockIdx.z;
  const int n_tiles = (p.Nkv + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(map_q);
    tma_prefetch_desc(map_k);
    tma_prefetch_desc(map_v);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  const float ip_scale = IP ? *p.ip_scale : 0.f;
  const bool ip = IP && ip_scale != 0.f;   // uniform over the CTA
  const int n_fills = n_tiles + (ip ? 1 : 0);  // ring fills: the text tiles, then the image tile

  auto load_kv = [&](int j) {  // thread 0
    const int s = j & 1;
    const bool image = IP && j == n_tiles;
    const CUtensorMap* mk = image ? map_k2 : map_k;
    const CUtensorMap* mv = image ? map_v2 : map_v;
    const int row = image ? 0 : j * BKV;
    mbar_arrive_expect_tx(&kv_full[s], 2 * TILE_BYTES);
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      tma_load_3d(sK + s * TILE_BYTES + a * ATOM_BYTES, mk, &kv_full[s], head * HD + a * 64, row, batch);
      tma_load_3d(sV + s * TILE_BYTES + a * ATOM_BYTES, mv, &kv_full[s], head * HD + a * 64, row, batch);
    }
  };
  if (threadIdx.x == 0) {
    if (IP) {
      tma_prefetch_desc(map_k2);
      tma_prefetch_desc(map_v2);
    }
    mbar_arrive_expect_tx(q_full, TILE_BYTES);
#pragma unroll
    for (int a = 0; a < NA; ++a) tma_load_3d(sQ + a * ATOM_BYTES, map_q, q_full, head * HD + a * 64, q0, batch);
    load_kv(0);
    if (n_fills > 1) load_kv(1);
  }

  const float c = p.scale_log2e;
  // accumulator fragment (m16n8): o[n][0..1] = (row lane / 4, cols 8 n + 2 (lane % 4) + {0, 1}), o[n][2..3] = row + 8
  float o[HD / 8][4];
#pragma unroll
  for (int n = 0; n < HD / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_base = smem_u32(sQ);
  const int qrow_ld = warp * 16 + (lane & 15);  // ldmatrix row of this lane for the A operand (Q)
  // S = Q K^T of one KV tile: 16 rows x 64 kv columns per warp; columns >= valid are set to -inf
  auto scores = [&](uint32_t k_base, int valid, float (&sc)[BKV / 8][4]) {
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      uint32_t a[4];
      ldmatrix_x4(q_base + tile_off(qrow_ld, 2 * kk + (lane >> 4)), a[0], a[1], a[2], a[3]);
#pragma unroll
      for (int n2 = 0; n2 < BKV / 16; ++n2) {  // two 8-column n tiles per ldmatrix.x4
        const int krow = n2 * 16 + (lane & 7) + ((lane >> 4) << 3);
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4(k_base + tile_off(krow, 2 * kk + ((lane >> 3) & 1)), b0, b1, b2, b3);
        mma_16816(sc[2 * n2], a, b0, b1);
        mma_16816(sc[2 * n2 + 1], a, b2, b3);
      }
    }
    if (valid < BKV) {
#pragma unroll
      for (int n = 0; n < BKV / 8; ++n) {
        const int col = n * 8 + 2 * (lane & 3);
        if (col >= valid) sc[n][0] = sc[n][2] = -INFINITY;
        if (col + 1 >= valid) sc[n][1] = sc[n][3] = -INFINITY;
      }
    }
  };
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int s = j & 1;
    mbar_wait(&kv_full[s], (j >> 1) & 1);
    const uint32_t k_base = smem_u32(sK + s * TILE_BYTES);
    const uint32_t v_base = smem_u32(sV + s * TILE_BYTES);
    float sc[BKV / 8][4];
    scores(k_base, p.Nkv - j * BKV, sc);  // columns past Nkv are padding (last tile only)
    // ---- online softmax (rows lane / 4 and lane / 4 + 8; the four lanes of a quad share a row) ----
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int n = 0; n < BKV / 8; ++n) mx = fmaxf(mx, fmaxf(sc[n][2 * h], sc[n][2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);  // finite: every tile holds at least one valid column
      alpha[h] = fast_exp2((m_run[h] - m_new) * c);
      m_run[h] = m_new;
    }
    float rs[2] = {0.f, 0.f};
    uint32_t pa[BKV / 8][2];  // P rounded to fp16, packed pairs in the accumulator layout
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float mc = m_run[h] * c;
        const float p0 = fast_exp2(sc[n][2 * h] * c - mc);
        const float p1 = fast_exp2(sc[n][2 * h + 1] * c - mc);
        rs[h] += p0 + p1;
        pa[n][h] = pack_half2(p0, p1);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + rs[h];  // per-lane partial; quad-reduced at the end
#pragma unroll
    for (int n = 0; n < HD / 8; ++n) {
      o[n][0] *= alpha[0];
      o[n][1] *= alpha[0];
      o[n][2] *= alpha[1];
      o[n][3] *= alpha[1];
    }
    // ---- O += P V: the m16n8 accumulators of kv columns [16 t, 16 t + 16) are the A fragment of k step t ----
#pragma unroll
    for (int t = 0; t < BKV / 16; ++t) {
      const uint32_t a[4] = {pa[2 * t][0], pa[2 * t][1], pa[2 * t + 1][0], pa[2 * t + 1][1]};
      const int vrow = t * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
#pragma unroll
      for (int d2 = 0; d2 < HD / 16; ++d2) {  // two 8-column d tiles per ldmatrix.x4.trans
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(v_base + tile_off(vrow, 2 * d2 + (lane >> 4)), b0, b1, b2, b3);
        mma_16816(o[2 * d2], a, b0, b1);
        mma_16816(o[2 * d2 + 1], a, b2, b3);
      }
    }
    __syncthreads();  // every warp is done with stage s
    if (threadIdx.x == 0 && j + 2 < n_fills) load_kv(j + 2);
  }

  float inv_l[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv_l[h] = 1.0f / l;
  }
  if (ip) {
    // ---- the image tile: one KV tile, so its max and sum are final before PV; a softmax of its own ----
    const int s = n_tiles & 1;
    mbar_wait(&kv_full[s], (n_tiles >> 1) & 1);
    const uint32_t v_base = smem_u32(sV + s * TILE_BYTES);
    float sc[BKV / 8][4];
    scores(smem_u32(sK + s * TILE_BYTES), p.Nkv2, sc);
    float mc[2], inv_l2[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int n = 0; n < BKV / 8; ++n) mx = fmaxf(mx, fmaxf(sc[n][2 * h], sc[n][2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      mc[h] = mx * c;  // finite: Nkv2 >= 1
    }
    float rs[2] = {0.f, 0.f};
    uint32_t pa[BKV / 8][2];
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float p0 = fast_exp2(sc[n][2 * h] * c - mc[h]);
        const float p1 = fast_exp2(sc[n][2 * h + 1] * c - mc[h]);
        rs[h] += p0 + p1;
        pa[n][h] = pack_half2(p0, p1);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = rs[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      inv_l2[h] = 1.0f / l;
    }
    // O2 = P V2 two d tiles at a time, over the k steps that hold valid image tokens (P and V2 are zero past Nkv2),
    // folded straight into o: o = O1 / l1 + s * O2 / l2
    const int k_steps = (p.Nkv2 + 15) / 16;
#pragma unroll
    for (int d2 = 0; d2 < HD / 16; ++d2) {
      float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int t = 0; t < BKV / 16; ++t) {
        if (t >= k_steps) break;
        const uint32_t a[4] = {pa[2 * t][0], pa[2 * t][1], pa[2 * t + 1][0], pa[2 * t + 1][1]};
        const int vrow = t * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(v_base + tile_off(vrow, 2 * d2 + (lane >> 4)), b0, b1, b2, b3);
        mma_16816(acc[0], a, b0, b1);
        mma_16816(acc[1], a, b2, b3);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          o[2 * d2 + i][e] = o[2 * d2 + i][e] * inv_l[e >> 1] + ip_scale * (acc[i][e] * inv_l2[e >> 1]);
    }
    inv_l[0] = inv_l[1] = 1.0f;  // o holds the output
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int qrow = q0 + warp * 16 + (lane >> 2) + 8 * h;
    if (qrow >= p.Nq) continue;
    __half* dst = p.out + (static_cast<size_t>(batch) * p.Nq + qrow) * p.ldo + head * HD + 2 * (lane & 3);
#pragma unroll
    for (int n = 0; n < HD / 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack_half2(o[n][2 * h] * inv_l[h], o[n][2 * h + 1] * inv_l[h]);
  }
}

template <int HD>
__global__ void __launch_bounds__(kThreads)
attn_kernel(const AttnParams p, const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
            const __grid_constant__ CUtensorMap map_v) {
  attn_body<HD, false>(p, &map_q, &map_k, &map_v, nullptr, nullptr);
}

template <int HD>
__global__ void __launch_bounds__(kThreads)
attn_ip_kernel(const AttnParams p, const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
               const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_k2,
               const __grid_constant__ CUtensorMap map_v2) {
  attn_body<HD, true>(p, &map_q, &map_k, &map_v, &map_k2, &map_v2);
}

// ---------------------------------------------------------------------------------------------------------------
// Head dim 64 (padded): warp-specialised wgmma kernel. One CTA = one 128-row query tile of one (batch, head), 384
// threads, 1 CTA / SM:
//   warpgroups 0, 1 : consumers; warpgroup g owns query rows [64 g, 64 g + 64). S = Q K^T is wgmma m64n128k16 with
//                     both operands in shared memory (K-major, 128B swizzle); the online softmax runs on the fp32
//                     accumulator, whose per-warp layout is the m16n8 fragment of the mma.sync kernel above (same
//                     rounding points); P rounded to fp16 is the register A operand of O += P V (wgmma m64n64k16,
//                     V an MN-major B operand).
//   warpgroup 2     : one thread issues TMA: Q once, then K / V as 128-row tiles into a W_STAGES-deep ring
//                     (full / empty mbarriers, no CTA-wide barrier in the loop).
// Each consumer issues S_j together with P_{j-1} V_{j-1} as one wgmma group, then runs the softmax of S_j. Two named
// barriers hand the tensor pipe back and forth between the warpgroups, so one warpgroup's softmax runs under the
// other's GEMMs. Every wgmma group is retired before the softmax: none stays in flight across the loop.
// ---------------------------------------------------------------------------------------------------------------
constexpr int W_BQ = 128;
constexpr int W_BKV = 128;
constexpr int W_STAGES = 4;
constexpr int W_THREADS = 384;
constexpr int W_KV_BYTES = 2 * ATOM_BYTES;  // one 128-row K or V tile: two 64-row TMA boxes
constexpr int W_SMEM_BYTES = 2 * ATOM_BYTES + W_STAGES * 2 * W_KV_BYTES + 1024 + 256;
static_assert(W_SMEM_BYTES <= 232448, "shared memory overflow");
constexpr int kTurnBar = 1;  // named barriers kTurnBar + g: warpgroup g may issue its wgmma group

// IP: the image tokens' K / V arrive as one more ring fill (64-row boxes, p.Nkv2 valid rows, TMA zero fill past
// them; the slot's rows 64..127 are left from an earlier fill or never written). S over that slot reads them but the
// mask replaces those columns, and PV runs over rows 0..63 only, which the fill wrote (zeros past Nkv2).
template <bool IP>
CFGPP_DEVICE void attn64_body(const AttnParams& p, const CUtensorMap* map_q, const CUtensorMap* map_k,
                              const CUtensorMap* map_v, const CUtensorMap* map_k2, const CUtensorMap* map_v2) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* sQ = smem;                            // [128 rows x 64]: warpgroup g reads atom g
  uint8_t* sK = sQ + 2 * ATOM_BYTES;             // W_STAGES x [128 rows x 64]
  uint8_t* sV = sK + W_STAGES * W_KV_BYTES;      // W_STAGES x [128 rows x 64]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + W_STAGES * W_KV_BYTES);
  uint64_t* full = q_full + 1;                   // [W_STAGES]
  uint64_t* empty = full + W_STAGES;             // [W_STAGES]: one arrive per consumer warp

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * W_BQ;
  const int head = blockIdx.y;
  const int batch = blockIdx.z;
  const int n_tiles = (p.Nkv + W_BKV - 1) / W_BKV;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < W_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  const float ip_scale = IP ? *p.ip_scale : 0.f;
  const bool ip = IP && ip_scale != 0.f;  // uniform over the CTA

  if (warp >= 8) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 256) {
      tma_prefetch_desc(map_q);
      tma_prefetch_desc(map_k);
      tma_prefetch_desc(map_v);
      if (IP) {
        tma_prefetch_desc(map_k2);
        tma_prefetch_desc(map_v2);
      }
      mbar_arrive_expect_tx(q_full, 2 * ATOM_BYTES);
      tma_load_3d(sQ, map_q, q_full, head * 64, q0, batch);
      tma_load_3d(sQ + ATOM_BYTES, map_q, q_full, head * 64, q0 + 64, batch);
      for (int f = 0; f < n_tiles + (IP ? 1 : 0); ++f) {
        const int s = f % W_STAGES;
        mbar_wait_nocall(&empty[s], ((f / W_STAGES) & 1) ^ 1);
        uint8_t* k_dst = sK + s * W_KV_BYTES;
        uint8_t* v_dst = sV + s * W_KV_BYTES;
        if (IP && f == n_tiles) {
          mbar_arrive_expect_tx(&full[s], 2 * ATOM_BYTES);
          tma_load_3d(k_dst, map_k2, &full[s], head * 64, 0, batch);
          tma_load_3d(v_dst, map_v2, &full[s], head * 64, 0, batch);
        } else {
          mbar_arrive_expect_tx(&full[s], 4 * ATOM_BYTES);
          for (int h = 0; h < 2; ++h) {
            tma_load_3d(k_dst + h * ATOM_BYTES, map_k, &full[s], head * 64, f * W_BKV + h * 64, batch);
            tma_load_3d(v_dst + h * ATOM_BYTES, map_v, &full[s], head * 64, f * W_BKV + h * 64, batch);
          }
        }
      }
    }
    return;
  }

  // ===================== consumers (warpgroups 0 and 1) =====================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  const float c = p.scale_log2e;
  // accumulator fragments: sc[8 n + e] / o[4 n + e] hold (row r, column 8 n + 2 (lane % 4) + e) for e < 2 and
  // (row r + 8, same column) for e >= 2, r = 16 (warp % 4) + lane / 4 of the warpgroup's 64 rows
  float sc[W_BKV / 2];
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  uint32_t pa[W_BKV / 4];  // P rounded to fp16: pa[2 n + h] packs sc[4 n + 2 h], sc[4 n + 2 h + 1]
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint64_t q_desc = make_wgmma_desc_sw128(smem_u32(sQ + wg * ATOM_BYTES));

  auto issue_s = [&](int s) {
    const uint64_t k_desc = make_wgmma_desc_sw128(smem_u32(sK + s * W_KV_BYTES));
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_f16<W_BKV>(sc, q_desc + 2 * k, k_desc + 2 * k, k != 0 ? 1u : 0u);
  };
  // acc += P V over the first ROWS rows of slot s
  auto issue_pv = [&](float (&acc)[32], int s, auto rows) {
    const uint64_t v_desc = make_wgmma_desc_sw128_mn(smem_u32(sV + s * W_KV_BYTES));
#pragma unroll
    for (int t = 0; t < decltype(rows)::value / 16; ++t) {
      const uint32_t a[4] = {pa[4 * t], pa[4 * t + 1], pa[4 * t + 2], pa[4 * t + 3]};
      wgmma_f16_rs_tb64(acc, a, v_desc + 128 * t, 1u);
    }
  };
  // online softmax of sc (columns >= valid set to -inf) against the running (m, l); rescales acc, writes pa
  auto softmax = [&](int valid, float (&m)[2], float (&l)[2], float (&acc)[32]) {
    if (valid < W_BKV) {
#pragma unroll
      for (int n = 0; n < W_BKV / 8; ++n) {
        const int col = n * 8 + 2 * (lane & 3);
        if (col >= valid) sc[4 * n] = sc[4 * n + 2] = -INFINITY;
        if (col + 1 >= valid) sc[4 * n + 1] = sc[4 * n + 3] = -INFINITY;
      }
    }
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int n = 0; n < W_BKV / 8; ++n) mx = fmaxf(mx, fmaxf(sc[4 * n + 2 * h], sc[4 * n + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx);  // finite: every tile holds at least one valid column
      alpha[h] = fast_exp2((m[h] - m_new) * c);
      m[h] = m_new;
    }
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int n = 0; n < W_BKV / 8; ++n) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float mc = m[h] * c;
        const float p0 = fast_exp2(sc[4 * n + 2 * h] * c - mc);
        const float p1 = fast_exp2(sc[4 * n + 2 * h + 1] * c - mc);
        rs[h] += p0 + p1;
        pa[2 * n + h] = pack_half2(p0, p1);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l[h] = l[h] * alpha[h] + rs[h];  // per-lane partial; quad-reduced at the end
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      acc[4 * n] *= alpha[0];
      acc[4 * n + 1] *= alpha[0];
      acc[4 * n + 2] *= alpha[1];
      acc[4 * n + 3] *= alpha[1];
    }
  };

  mbar_wait_nocall(q_full, 0);
  if (wg == 1) named_bar_arrive(kTurnBar, 256);  // warpgroup 0 issues first
  // Step 0 issues S_0; step j in [1, n_tiles) issues S_j and P_{j-1} V_{j-1} as one group; the last step P V of the
  // last tile. A warpgroup issues a step once the other has issued its previous one. No wgmma sits on a branch (a
  // wgmma under a condition ptxas cannot prove uniform makes it serialise every wgmma of the kernel).
  constexpr std::integral_constant<int, W_BKV> kAllRows{};
  mbar_wait_nocall(&full[0], 0);
  named_bar_sync(kTurnBar + wg, 256);
  wgmma_fence();
  issue_s(0);
  wgmma_commit();
  named_bar_arrive(kTurnBar + (wg ^ 1), 256);
  wgmma_wait<0>();
  fence_acc(sc);
  softmax(p.Nkv, m_run, l_run, o);  // columns past Nkv: padding (last tile only)
  for (int j = 1; j < n_tiles; ++j) {
    const int s = j % W_STAGES;
    const int sp = (j - 1) % W_STAGES;
    mbar_wait_nocall(&full[s], (j / W_STAGES) & 1);
    named_bar_sync(kTurnBar + wg, 256);
    wgmma_fence();
    issue_s(s);
    issue_pv(o, sp, kAllRows);
    wgmma_commit();
    named_bar_arrive(kTurnBar + (wg ^ 1), 256);
    wgmma_wait<0>();
    fence_acc(sc);
    fence_acc(o);
    fence_acc(pa);
    if (lane == 0) mbar_arrive(&empty[sp]);
    softmax(p.Nkv - j * W_BKV, m_run, l_run, o);
  }
  const int s_last = (n_tiles - 1) % W_STAGES;
  named_bar_sync(kTurnBar + wg, 256);
  wgmma_fence();
  issue_pv(o, s_last, kAllRows);
  wgmma_commit();
  if (wg == 0) named_bar_arrive(kTurnBar + 1, 256);  // warpgroup 1's last sync; its own first arrive balances ours
  wgmma_wait<0>();
  fence_acc(o);
  fence_acc(pa);
  if (lane == 0) mbar_arrive(&empty[s_last]);

  float inv_l[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv_l[h] = 1.0f / l;
  }
  if constexpr (IP) {
    // ---- the image tile: one ring fill, a softmax of its own (max and sum final before PV). It is computed at
    // s = 0 as well (a branch around it would serialise the wgmmas) and dropped by the select below. ----
    const int s = n_tiles % W_STAGES;
    mbar_wait_nocall(&full[s], (n_tiles / W_STAGES) & 1);
    wgmma_fence();
    issue_s(s);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(sc);
    float m2[2] = {-INFINITY, -INFINITY}, l2[2] = {0.f, 0.f};
    float o2[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o2[i] = 0.f;
    softmax(p.Nkv2, m2, l2, o2);
    wgmma_fence();
    issue_pv(o2, s, std::integral_constant<int, 64>{});  // the rows this fill wrote; P and V2 are zero past Nkv2
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(o2);
    fence_acc(pa);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = l2[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      l2[h] = 1.0f / l;
    }
    // o = O1 / l1 + s * O2 / l2, rounded once below; s = 0 keeps the plain kernel's o / l1
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float fold = o[i] * inv_l[(i >> 1) & 1] + ip_scale * (o2[i] * l2[(i >> 1) & 1]);
      o[i] = ip ? fold : o[i];
    }
    if (ip) inv_l[0] = inv_l[1] = 1.0f;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int qrow = q0 + warp * 16 + (lane >> 2) + 8 * h;  // warp = 4 wg + warp % 4
    if (qrow >= p.Nq) continue;
    __half* dst = p.out + (static_cast<size_t>(batch) * p.Nq + qrow) * p.ldo + head * 64 + 2 * (lane & 3);
#pragma unroll
    for (int n = 0; n < 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack_half2(o[4 * n + 2 * h] * inv_l[h], o[4 * n + 2 * h + 1] * inv_l[h]);
  }
}

__global__ void __launch_bounds__(W_THREADS, 1)
attn64_kernel(const AttnParams p, const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
              const __grid_constant__ CUtensorMap map_v) {
  attn64_body<false>(p, &map_q, &map_k, &map_v, nullptr, nullptr);
}

__global__ void __launch_bounds__(W_THREADS, 1)
attn64_ip_kernel(const AttnParams p, const __grid_constant__ CUtensorMap map_q,
                 const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                 const __grid_constant__ CUtensorMap map_k2, const __grid_constant__ CUtensorMap map_v2) {
  attn64_body<true>(p, &map_q, &map_k, &map_v, &map_k2, &map_v2);
}

void launch64(const AttnOp& op, cudaStream_t stream) {
  dim3 grid((op.p.Nq + W_BQ - 1) / W_BQ, op.p.H, op.p.B);
  if (op.p.ip_scale)
    launch_pdl(attn64_ip_kernel, grid, dim3(W_THREADS), W_SMEM_BYTES, stream, op.p, op.map_q, op.map_k, op.map_v,
               op.map_k2, op.map_v2);
  else
    launch_pdl(attn64_kernel, grid, dim3(W_THREADS), W_SMEM_BYTES, stream, op.p, op.map_q, op.map_k, op.map_v);
}

CUtensorMap make_head_map(const __half* base, int ld, int B, int N, int cols) {
  uint64_t dims[3] = {(uint64_t)cols, (uint64_t)N, (uint64_t)B};
  uint64_t strides[2] = {(uint64_t)ld * 2, (uint64_t)N * ld * 2};
  uint32_t box[3] = {64, 64, 1};
  return make_tmap_f16(base, 3, dims, strides, box);
}

template <int HD>
void configure_one() {
  CFGPP_CHECK_CUDA(cudaFuncSetAttribute(attn_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        ACfg<HD>::SMEM_BYTES));
  CFGPP_CHECK_CUDA(cudaFuncSetAttribute(attn_ip_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        ACfg<HD>::SMEM_BYTES));
}

template <int HD>
void launch(const AttnOp& op, cudaStream_t stream) {
  dim3 grid((op.p.Nq + BQ - 1) / BQ, op.p.H, op.p.B);
  if (op.p.ip_scale)
    launch_pdl(attn_ip_kernel<HD>, grid, dim3(kThreads), ACfg<HD>::SMEM_BYTES, stream, op.p, op.map_q, op.map_k,
               op.map_v, op.map_k2, op.map_v2);
  else
    launch_pdl(attn_kernel<HD>, grid, dim3(kThreads), ACfg<HD>::SMEM_BYTES, stream, op.p, op.map_q, op.map_k,
               op.map_v);
}

}  // namespace

int attn_padded_head_dim(int head_dim) { return ((head_dim + 63) / 64) * 64; }

AttnOp make_attn_op(const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, __half* out,
                    int ldo, int B, int H, int Nq, int Nkv, int head_dim) {
  AttnOp op{};
  CFGPP_REQUIRE(Nkv >= 1 && Nq >= 1, "empty attention");
  CFGPP_REQUIRE(ldo % 8 == 0, "ldo must be a multiple of 8");
  CFGPP_REQUIRE(head_dim >= 8 && head_dim <= 192, "attention supports head_dim <= 192");
  const int hdp = attn_padded_head_dim(head_dim);
  op.hd_pad = hdp;
  op.head_dim = head_dim;
  op.p.B = B; op.p.H = H; op.p.Nq = Nq; op.p.Nkv = Nkv; op.p.ldo = ldo; op.p.out = out;
  op.p.scale_log2e = (1.0f / sqrtf(static_cast<float>(head_dim))) * 1.4426950408889634f;
  op.map_q = make_head_map(q, ldq, B, Nq, H * hdp);
  op.map_k = make_head_map(k, ldk, B, Nkv, H * hdp);
  op.map_v = make_head_map(v, ldv, B, Nkv, H * hdp);
  return op;
}

AttnOp make_attn_ip_op(const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, const __half* k2,
                       int ldk2, const __half* v2, int ldv2, int Nkv2, const float* ip_scale, __half* out, int ldo,
                       int B, int H, int Nq, int Nkv, int head_dim) {
  CFGPP_REQUIRE(Nkv2 >= 1 && Nkv2 <= 64, "the image segment holds 1..64 tokens");
  CFGPP_REQUIRE(ip_scale != nullptr, "the image segment needs its scale word");
  AttnOp op = make_attn_op(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Nq, Nkv, head_dim);
  op.p.Nkv2 = Nkv2;
  op.p.ip_scale = ip_scale;
  op.map_k2 = make_head_map(k2, ldk2, B, Nkv2, H * op.hd_pad);
  op.map_v2 = make_head_map(v2, ldv2, B, Nkv2, H * op.hd_pad);
  return op;
}

void attn_configure() {
  static bool done = false;
  if (done) return;
  CFGPP_CHECK_CUDA(cudaFuncSetAttribute(attn64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, W_SMEM_BYTES));
  CFGPP_CHECK_CUDA(cudaFuncSetAttribute(attn64_ip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, W_SMEM_BYTES));
  configure_one<128>();
  configure_one<192>();
  done = true;
}

void run_attn_op(const AttnOp& op, cudaStream_t stream) {
  attn_configure();
  switch (op.hd_pad) {
    case 64: return launch64(op, stream);
    case 128: return launch<128>(op, stream);
    case 192: return launch<192>(op, stream);
    default: throw Error(-1, "unsupported padded head dim");
  }
}

}  // namespace cfgpp
