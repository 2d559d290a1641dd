// cfgpp_b200 — persistent, warp-specialised wgmma GEMM / implicit-GEMM conv3x3 kernel for sm_90a.
// See gemm.cuh for the operator contract. Structure per CTA (384 threads = 3 warpgroups, 1 CTA / SM, persistent over
// tiles):
//   warpgroups 0, 1 : MMA + epilogue arithmetic. Warpgroup g owns rows [64 g, 64 g + 64) of the 128 x BN tile: wgmma
//                     m64nBNk16 from the shared-memory ring into a register accumulator, then bias / addend / GEGLU /
//                     LN-fold -> fp16 into a swizzled smem staging tile, from vectors already in shared memory; then
//                     straight on to the next tile's main loop. Warp w of the group owns 16 rows end to end.
//   warp 8, lane 0  : TMA producer (A tile 128x64, B tile BNx64 per stage, 128B swizzle, mbarrier complete_tx).
//   warps 9 .. 11   : epilogue service, off the MMA warps' critical path: they stage the per-tile vectors (bias,
//                     time-embedding row, LN-fold s_n / t_n and the fold's per-row sums) two tiles ahead from global
//                     memory, and lanes 0..7 of warp 9 issue the staged tile's TMA stores, wait for their read-out and
//                     prefetch the next tile's residual into the staging tile.
// Warpgroup 2 hands registers to the MMA warpgroups (setmaxnreg), which hold up to 128 fp32 accumulator registers per
// thread. Pipeline: smem ring full/empty (TMA <-> MMA); staging tile staged/free (MMA <-> store lanes); vector buffers
// vec per parity (service warps -> MMA; the tile's staged arrival hands the buffer back).
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "gemm.cuh"

namespace cfgpp {

void gemm_configure();

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kThreads = 384;
constexpr int kEpiWarps = 8;      // warps 0..7: MMA + epilogue (warpgroups 0 and 1)
constexpr int kProducerWarp = 8;
constexpr int kSvcWarp0 = 9;      // warps 9..11: epilogue service (vector staging, TMA stores)
constexpr int kSvcThreads = 3 * 32;
constexpr int A_BYTES = BM * BK * 2;
constexpr int kSkMaxCtas = 256;            // stream-K: flags[c] arrivals, flags[kSkDoneOffset + c] consumers
constexpr int kSkDoneOffset = kSkMaxCtas;

template <int BN, bool GEGLU>
struct Cfg {
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // output columns of a tile and its smem staging area: OUT_N / 32 sub-tiles of [128 rows x 64 B], 64B swizzle
  static constexpr int OUT_N = GEGLU ? BN / 2 : BN;
  static constexpr int EPI_SUB = OUT_N / 32;
  static constexpr int EPI_SUB_BYTES = BM * 64;
  static constexpr int EPI_BYTES = EPI_SUB * EPI_SUB_BYTES;
  static constexpr int STAGES = GEGLU ? 3 : (BN == 256 ? 3 : (BN == 160 ? 4 : 5));
  // per-tile vectors staged for the epilogue: bias + time-embedding row (fp16), LayerNorm-fold s_n / t_n (fp32), and
  // the LayerNorm fold's per-row (sum, sum of squares) of the tile's 128 rows (float2)
  static constexpr int VEC_ONE = 2 * 256 * 2 + 2 * 256 * 4 + BM * 8;
  static constexpr int VEC_BYTES = 2 * VEC_ONE;  // double-buffered by epilogue-tile parity
  static constexpr int SMEM_BYTES =
      STAGES * STAGE_BYTES + EPI_BYTES + VEC_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB shared memory of an SM");
  static constexpr int ACC = BN / 2;  // fp32 accumulator registers per thread (m64 x BN over 128 threads)
};

// SCALED: the scaled-residual epilogue (GemmParams::res_scale), a kernel of its own so that the production epilogues
// compile exactly as they would without it
template <int BN, bool GEGLU, bool SCALED = false>
__global__ void __launch_bounds__(kThreads, 1)
gemm_kernel(const GemmParams p, const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_a2,
            const __grid_constant__ CUtensorMap map_b, const __grid_constant__ CUtensorMap map_out,
            const __grid_constant__ CUtensorMap map_res) {
  using C = Cfg<BN, GEGLU>;
  extern __shared__ uint8_t smem_raw[];
  // 1024B alignment (required by the 128B swizzle atoms) in the shared address space
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);

  uint8_t* epi_smem = smem + C::STAGES * C::STAGE_BYTES;
  // 2 x { bias[256] fp16, temb[256] fp16, ln_s[256] fp32, ln_t[256] fp32, ln_sum[128] float2 }
  uint8_t* vec_smem = epi_smem + C::EPI_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_smem + C::EPI_BYTES + C::VEC_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + C::STAGES;
  uint64_t* res_bar = bars + 2 * C::STAGES;  // [kEpiWarps]: the residual sub-blocks of each epilogue warp's 16 rows
  // [2] by epilogue-tile parity: every MMA thread has written its part of the staging tile and read the tile's vectors
  // (two barriers, so a service warp that lags one tile behind can never mistake the next phase for the one it waits on)
  uint64_t* staged_bar = res_bar + kEpiWarps;
  uint64_t* free_bar = staged_bar + 2;  // the store lanes have read the staging tile out (and issued the next residual)
  uint64_t* vec_bar = free_bar + 1;     // [2] by parity: the service warps have staged that buffer's vectors

  const int warp_idx = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);  // provably warp-uniform
  const int lane = threadIdx.x & 31;
  unsigned long long* tl = p.timeline ? p.timeline + static_cast<size_t>(blockIdx.x) * 16 : nullptr;
#define TL(slot) do { if (tl) tl[slot] = globaltimer_ns(); } while (0)
  if (threadIdx.x == 0) TL(0);
  const int cta_id = blockIdx.x;
  const int num_ctas = gridDim.x;

  if (warp_idx == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_a2);
    tma_prefetch_desc(&map_b);
    tma_prefetch_desc(&map_out);
    tma_prefetch_desc(&map_res);
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kEpiWarps);  // one arrive per consumer warp once its wgmmas on the stage retired
    }
    for (int i = 0; i < kEpiWarps; ++i) mbar_init(&res_bar[i], 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&staged_bar[i], kEpiWarps * 32);
      mbar_init(&vec_bar[i], kSvcThreads);
    }
    mbar_init(free_bar, kEpiWarps);  // one store lane per epilogue warp's slab
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();  // the next kernel may start its prologue on SMs this grid leaves
  pdl_wait();               // everything above overlapped the previous kernel's tail; its outputs are needed below
  if (threadIdx.x == 0) TL(2);

  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const int nkb = p.num_k_blocks;
  auto tile_m_blk = [&](int tile) { return p.raster ? tile / p.num_n_blocks : tile % p.num_m_blocks; };
  auto tile_n_blk = [&](int tile) { return p.raster ? tile % p.num_n_blocks : tile / p.num_m_blocks; };

  // ---- work schedule: "stream-K for the remainder" -------------------------------------------------------------
  // D = the tiles that fill whole rounds over the CTAs are walked data-parallel (tile = cta + r * ctas); the
  // R = T mod ctas left-over tiles would cost a full extra round with most CTAs idle, so their R * nkb k-blocks are
  // split evenly over ALL CTAs instead: CTA c owns the contiguous unit range [c U / P, (c + 1) U / P) of the linearised
  // (tile, k-block) space — at most two pieces, of two adjacent tiles. The piece that contains a tile's LAST k-block
  // finishes the tile: the fp32 partial accumulators the other pieces parked in the workspace are summed in a fixed
  // order (deterministic) into its register accumulator before its main loop, and the normal epilogue follows. All
  // CTAs of the grid are co-resident (grid <= SMs, one CTA per SM; a dependent grid is only scheduled after every CTA
  // of this one has started), so the spin-wait on a peer's flag cannot deadlock; a waits-for edge always points at a
  // lower CTA's FIRST item.
  constexpr int kItemFull = 0, kItemPart = 1, kItemFin = 2;
  struct Item {
    int tile, kb0, kb1, kind, c_first;
  };
  int sk_r = 0;  // R
  long sk_units = 0;
  if (p.sk_ws != nullptr && num_tiles % num_ctas != 0) {
    sk_r = num_tiles % num_ctas;
    sk_units = static_cast<long>(sk_r) * nkb;
  }
  const int dp_tiles = num_tiles - sk_r;
  auto sk_u0 = [&](int c) { return static_cast<int>(sk_units * c / num_ctas); };
  // A CTA's stream-K share is at most one non-finishing piece (`sk_first`, walked FIRST so that its partial is
  // published while everybody still has main-loop work) and at most one finishing piece (`sk_late`, walked just
  // before the last data-parallel tile — or last when there is only one — so that the flag wait is rarely exposed).
  Item sk_first{}, sk_late{};
  int n_first = 0, n_late = 0;
  if (sk_r > 0) {
    const int u0 = sk_u0(cta_id), u1 = sk_u0(cta_id + 1);
    if (u1 > u0) {
      const int s0 = u0 / nkb;
      const int e0 = (u1 < (s0 + 1) * nkb) ? u1 : (s0 + 1) * nkb;
      auto make = [&](int s, int b, int e) {  // units [b, e) of stream-K tile s
        Item it;
        it.tile = dp_tiles + s;
        it.kb0 = b - s * nkb;
        it.kb1 = e - s * nkb;
        it.c_first = cta_id;
        if (it.kb1 < nkb) {
          it.kind = kItemPart;
        } else if (it.kb0 == 0) {
          it.kind = kItemFull;
        } else {
          it.kind = kItemFin;
          int c = cta_id;
          while (c > 0 && sk_u0(c) > s * nkb) --c;  // the CTA whose range holds the tile's first k-block
          it.c_first = c;
        }
        return it;
      };
      if (u1 > e0) {  // head of the next tile: never finishing
        sk_first = make(s0 + 1, e0, u1);
        n_first = 1;
      }
      const Item a = make(s0, u0, e0);
      if (a.kind == kItemPart) {
        sk_first = a;  // (a piece strictly inside one tile: then there is no second piece)
        n_first = 1;
      } else {
        sk_late = a;
        n_late = 1;
      }
    }
  }
  const int n_dp = (dp_tiles > cta_id) ? (dp_tiles - cta_id + num_ctas - 1) / num_ctas : 0;
  const int n_items = n_first + n_late + n_dp;
  const int late_pos = n_first + (n_dp >= 2 ? n_dp - 1 : n_dp);
  auto item_at = [&](int i) {
    if (i < n_first) return sk_first;
    if (n_late && i == late_pos) return sk_late;
    Item it;
    it.tile = cta_id + (i - n_first - ((n_late && i > late_pos) ? 1 : 0)) * num_ctas;
    it.kb0 = 0;
    it.kb1 = nkb;
    it.kind = kItemFull;
    it.c_first = cta_id;
    return it;
  };
  constexpr unsigned kSkArrivals = kEpiWarps;  // warps that publish / consume one CTA's partial
  // partial accumulator of CTA c: [BN / 4 register pairs][256 consumer threads] float2 (the register fragment order)
  auto sk_ws = [&](int c) { return p.sk_ws + static_cast<size_t>(c) * (static_cast<size_t>(BM) * BN); };

  // ---- epilogue tiles: every item except the stream-K pieces that only park a partial ----------------------------
  static_assert((2 * C::STAGES + kEpiWarps + 5) * 8 <= 256, "barrier area");
  auto next_epi_item = [&](int from) {
    int i = from;
    while (i < n_items && item_at(i).kind == kItemPart) ++i;
    return i;
  };
  const bool full_res = (p.addend != nullptr) && (p.add_rows_per_group <= 1);
  // a time-embedding row is staged in shared memory when all of the tile's rows belong to one sample
  auto temb_staged_for = [&](int m_blk) {
    const int m_first = m_blk * BM;
    const int m_last = (m_first + BM - 1 < p.M ? m_first + BM - 1 : p.M - 1);
    return p.addend != nullptr && !full_res && (m_first < p.M) &&
           (m_first / p.add_rows_per_group == m_last / p.add_rows_per_group);
  };
  auto vec_bias = [&](int parity) { return reinterpret_cast<__half*>(vec_smem + parity * C::VEC_ONE); };  // [256]
  auto vec_temb = [&](int parity) { return vec_bias(parity) + 256; };                                       // [256]
  auto vec_lns = [&](int parity) { return reinterpret_cast<float*>(vec_temb(parity) + 256); };             // [256]
  auto vec_lnt = [&](int parity) { return vec_lns(parity) + 256; };                                        // [256]
  auto vec_lnsum = [&](int parity) { return reinterpret_cast<float2*>(vec_lnt(parity) + 256); };           // [128]
  // residual sub-blocks of epilogue warp w's 16 rows, into its slab of the staging tile (one lane)
  auto issue_residual = [&](int tile, int w) {
    const int m_blk = tile_m_blk(tile);
    const int n_blk = tile_n_blk(tile);
    mbar_arrive_expect_tx(&res_bar[w], C::EPI_SUB * 16 * 64);
#pragma unroll 1
    for (int j = 0; j < C::EPI_SUB; ++j)
      tma_load_2d(epi_smem + w * 16 * 64 + j * C::EPI_SUB_BYTES, &map_res, &res_bar[w], n_blk * C::OUT_N + j * 32,
                  m_blk * BM + w * 16);
  };

  if (warp_idx >= kEpiWarps) {
    setmaxnreg_dec<40>();
    if (warp_idx >= kSvcWarp0) {
      // ===================== epilogue service =====================
      const int st = threadIdx.x - kSvcWarp0 * 32;  // 0 .. kSvcThreads - 1
      // Stage the vectors of the tile's epilogue into buffer `parity`: bias (and, when all 128 rows belong to one
      // sample, its time-embedding row), the fold's s_n / t_n, and the rows' (sum, sum of squares) from the producer's
      // per-N-block partials, summed in a fixed order.
      auto stage_vectors = [&](int tile, int parity) {
        const int m_blk = tile_m_blk(tile);
        const int n_blk = tile_n_blk(tile);
        __half* s_bias = vec_bias(parity);
        __half* s_temb = vec_temb(parity);
        float* s_lns = vec_lns(parity);
        float* s_lnt = vec_lnt(parity);
        const bool temb = temb_staged_for(m_blk);
        const __half* temb_row = p.addend + (temb ? static_cast<size_t>(m_blk * BM / p.add_rows_per_group) * p.ld_add : 0);
        const int ncols = GEGLU ? BN : C::OUT_N;  // GEGLU stages value + gate biases (packed alike)
        const int n_base = n_blk * BN;
        for (int c = st; c < ncols; c += kSvcThreads) {
          const int n = n_base + c;
          const bool ok = n < p.N;
          s_bias[c] = (p.bias && ok) ? p.bias[n] : __float2half(0.f);
          if (temb) s_temb[c] = ok ? temb_row[n] : __float2half(0.f);
          if (p.stats_in) {
            s_lns[c] = ok ? p.ln_s[n] : 0.f;
            s_lnt[c] = ok ? p.ln_t[n] : 0.f;
          }
        }
        if (p.stats_in) {
          float2* s_sum = vec_lnsum(parity);
          for (int r = st; r < BM; r += kSvcThreads) {
            const int m = m_blk * BM + r;
            if (m >= p.M) continue;
            float sx = 0.f, sxx = 0.f;
            for (int i = 0; i < p.ln_parts; ++i) {
              const float2 v = *reinterpret_cast<const float2*>(p.stats_in + (static_cast<size_t>(i) * p.M + m) * 2);
              sx += v.x;
              sxx += v.y;
            }
            s_sum[r] = make_float2(sx, sxx);
          }
        }
        mbar_arrive(&vec_bar[parity]);
      };
      const int i0 = next_epi_item(0);
      const int i1 = i0 < n_items ? next_epi_item(i0 + 1) : n_items;
      if (full_res && warp_idx == kSvcWarp0 && lane < kEpiWarps && i0 < n_items) issue_residual(item_at(i0).tile, lane);
      if (i0 < n_items) stage_vectors(item_at(i0).tile, 0);
      if (i1 < n_items) stage_vectors(item_at(i1).tile, 1);
      int ahead = i1 < n_items ? next_epi_item(i1 + 1) : n_items;  // the epilogue tile two after the current one
      int e = 0;                                                    // epilogue tiles done
      for (int i = i0; i < n_items; ++e) {
        const int nx = next_epi_item(i + 1);
        mbar_wait_nocall(&staged_bar[e & 1], (e >> 1) & 1);
        if (warp_idx == kSvcWarp0 && lane < kEpiWarps) {
          if (lane == 0) TL(14);
          // lane w stores epilogue warp w's [16 x OUT_N] slab, then refills it with the next tile's residual
          const int tile = item_at(i).tile;
          const int m_blk = tile_m_blk(tile);
          const int n_blk = tile_n_blk(tile);
#pragma unroll 1
          for (int j = 0; j < C::EPI_SUB; ++j)
            tma_store_2d(&map_out, epi_smem + lane * 16 * 64 + j * C::EPI_SUB_BYTES, n_blk * C::OUT_N + j * 32,
                         m_blk * BM + lane * 16);
          tma_store_commit();
          if (lane == 0) {
            if (e == 0) TL(8);
            TL(10);
          }
          tma_store_wait_read0();
          if (full_res && nx < n_items) issue_residual(item_at(nx).tile, lane);
          mbar_arrive(free_bar);
          if (lane == 0) TL(15);
        }
        if (ahead < n_items) {  // the MMA threads are done with buffer e & 1: refill it for tile e + 2
          stage_vectors(item_at(ahead).tile, e & 1);
          ahead = next_epi_item(ahead + 1);
        }
        i = nx;
      }
      if (warp_idx == kSvcWarp0 && lane < kEpiWarps) tma_store_wait0();
      if (warp_idx == kSvcWarp0 && lane == 0) TL(11);
    } else if (lane == 0) {
      // ===================== TMA producer =====================
      int stage = 0;
      uint32_t phase = 0;
      for (int item_i = 0; item_i < n_items; ++item_i) {
        const Item item = item_at(item_i);
        const int tile = item.tile;
        const int m_blk = tile_m_blk(tile);
        const int n_blk = tile_n_blk(tile);
        const int m0 = m_blk * BM;
        int img = 0, h0 = 0, w0 = 0;
        if (p.conv) {
          const int hw = p.H * p.W;
          img = m0 / hw;
          const int r = m0 - img * hw;
          h0 = r / p.W;
          w0 = r - h0 * p.W;
        }
        for (int kb = item.kb0; kb < item.kb1; ++kb) {
          mbar_wait_nocall(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * C::STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          if (p.conv) {
            const int tap = kb / p.cpb;
            const int cb = kb - tap * p.cpb;
            const int kh = tap / 3, kw = tap - kh * 3;
            if (p.conv_im2col)  // the walk starts at the tile's first output pixel; the tap is the load's offset
              tma_load_im2col_4d(sa, &map_a, &full_bar[stage], cb * BK, w0 * p.conv_stride - p.conv_pad,
                                 h0 * p.conv_stride - p.conv_pad, img, static_cast<uint16_t>(kw),
                                 static_cast<uint16_t>(kh));
            else
              tma_load_4d(sa, &map_a, &full_bar[stage], cb * BK, w0 * p.conv_stride + kw - p.conv_pad,
                          h0 * p.conv_stride + kh - p.conv_pad, img);
          } else {
            const int k0 = kb * BK;
            if (k0 < p.k_split)
              tma_load_2d(sa, &map_a, &full_bar[stage], k0, m0);
            else
              tma_load_2d(sa, &map_a2, &full_bar[stage], k0 - p.k_split, m0);
          }
          tma_load_2d(sb, &map_b, &full_bar[stage], kb * BK, n_blk * BN);
          if (++stage == C::STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ===================== MMA + epilogue (warpgroups 0 and 1) =====================
    // Register fragment of the m64nBN accumulator: acc[4 i + e] is (row r0, column 8 i + 2 (lane % 4) + e),
    // acc[4 i + 2 + e] is (row r0 + 8, same column); r0 = 64 g + 16 (warp % 4) + lane / 4.
    const int wg = warp_idx >> 2;
    const int wq = warp_idx & 3;
    const int slab_row = wg * 64 + wq * 16;       // first tile row of this warp
    const int r0 = slab_row + (lane >> 2);        // this thread's two rows: r0, r0 + 8
    const int cq = 2 * (lane & 3);                // column offset inside an 8-column group
    const int etid = threadIdx.x;                 // 0..255
    const bool leader = (threadIdx.x == 0);
    uint64_t* my_res_bar = &res_bar[warp_idx];
    // byte offset of (tile row r, 8-column group q of a 32-column sub-tile) in the 64B-swizzled staging sub-tile
    auto stage_off = [&](int r, int q) { return r * 64 + ((q ^ ((r >> 1) & 3)) << 4) + (lane & 3) * 4; };
    int ep = 0;  // epilogue tiles done
    int res_uses = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[C::ACC];

    // Stream-K fix-up: the partial accumulators the other CTAs parked for this CTA's finishing piece are summed
    // (fixed order) into the registers its main loop then accumulates on top of.
    auto sk_preload = [&]() {
      auto contributes = [&](int c) { return sk_u0(c + 1) > sk_u0(c); };
      if (lane == 0) {  // acquire: every warp of every contributing CTA has published its partial
        for (int c = sk_late.c_first; c < cta_id; ++c) {
          if (!contributes(c)) continue;
          unsigned seen;
          const long long t0 = clock64();
          do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(p.sk_flags + c) : "memory");
            if (seen < kSkArrivals) __nanosleep(32);
            if (clock64() - t0 > 4000000000LL) __trap();  // a peer that never publishes is a scheduling bug
          } while (seen < kSkArrivals);
        }
      }
      __syncwarp();  // the other lanes' partial loads (L2, __ldcg) are ordered after lane 0's acquire
      // the first contributor's partial is assigned, the others are added: a select between the two would keep the
      // previous item's accumulator live through the loads
      int c0 = sk_late.c_first;
      while (!contributes(c0)) ++c0;  // the piece holding the tile's first k-block always contributes
      auto add_partial = [&](int c, auto assign_c) {
        constexpr bool ASSIGN = decltype(assign_c)::value;
        const float2* src = reinterpret_cast<const float2*>(sk_ws(c)) + etid;
#pragma unroll
        for (int i = 0; i < C::ACC / 2; ++i) {
          const float2 f = __ldcg(src + i * 256);
          acc[2 * i] = ASSIGN ? f.x : acc[2 * i] + f.x;
          acc[2 * i + 1] = ASSIGN ? f.y : acc[2 * i + 1] + f.y;
          // at most 8 loads in flight: hoisting all of them (BN = 256: 128 registers on top of the 128 of the
          // accumulator) made ptxas spill
          if (i % 8 == 7) asm volatile("" ::: "memory");
        }
      };
      add_partial(c0, std::true_type{});
      for (int c = c0 + 1; c < cta_id; ++c)
        if (contributes(c)) add_partial(c, std::false_type{});
      __syncwarp();
      if (lane == 0) {
        // this warp has consumed the partials: the last of the kSkArrivals consumers re-arms the contributor's flag,
        // so the buffers are back in their initial state when the kernel ends (CUDA-graph replays bake the arguments,
        // an epoch counter is not an option)
        for (int c = sk_late.c_first; c < cta_id; ++c) {
          if (!contributes(c)) continue;
          const unsigned old = atomicAdd(p.sk_flags + kSkDoneOffset + c, 1u);
          if (old == kSkArrivals - 1) {
            p.sk_flags[kSkDoneOffset + c] = 0u;
            p.sk_flags[c] = 0u;
          }
        }
      }
      __syncwarp();
    };

    for (int it = 0; it < n_items; ++it) {
      const Item item = item_at(it);
      const int tile = item.tile;
      if (leader && ep == 1) TL(6);
      // ---- main loop: wgmma over the smem ring, one k-block kept in flight ----
      // a finishing stream-K piece starts from the other pieces' partial sum, every other item from zero (scale-d 0)
      const bool preloaded = item.kind == kItemFin;
      if (preloaded) sk_preload();
      for (int kb = item.kb0; kb < item.kb1; ++kb) {
        mbar_wait_nocall(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * C::STAGE_BYTES) + wg * (64 * 128);
        const uint32_t b_addr = smem_u32(smem + stage * C::STAGE_BYTES) + A_BYTES;
        const uint64_t a_desc = make_wgmma_desc_sw128(a_addr);
        const uint64_t b_desc = make_wgmma_desc_sw128(b_addr);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_f16<BN>(acc, a_desc + 2 * k, b_desc + 2 * k, (preloaded || kb != item.kb0 || k != 0) ? 1u : 0u);
        wgmma_commit();
        // Retire the k-block before the next one (keeping one group in flight across iterations makes ptxas serialise
        // every wgmma); the producer is STAGES - 1 loads ahead, so only the tensor pipe's drain is exposed.
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == C::STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      fence_acc(acc);

      if (item.kind == kItemPart) {
        // ---- stream-K piece that does not finish its tile: park the raw fp32 accumulator, publish, move on ----
        // float2 pair i of thread t at [i][t]: one STG.64 of the warp writes 256 contiguous bytes
        float2* dst = reinterpret_cast<float2*>(sk_ws(cta_id)) + etid;
#pragma unroll
        for (int i = 0; i < C::ACC / 2; ++i) dst[i * 256] = make_float2(acc[2 * i], acc[2 * i + 1]);
        __syncwarp();  // the warp's stores happen-before lane 0's release below (barrier + cumulativity)
        if (lane == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p.sk_flags + cta_id) : "memory");
        __syncwarp();
        continue;
      }
      const int m_blk = tile_m_blk(tile);
      const int n_blk = tile_n_blk(tile);
      const int mrow[2] = {m_blk * BM + r0, m_blk * BM + r0 + 8};
      const int vb = ep & 1;
      if (leader) {
        if (ep == 0) TL(5);
        TL(7);
      }
      const __half* s_bias = vec_bias(vb);
      const __half* s_temb = vec_temb(vb);
      const float* s_lns = vec_lns(vb);
      const float* s_lnt = vec_lnt(vb);
      const __half* add_rows[2] = {nullptr, nullptr};  // per-sample row broadcast (ResnetBlock2D time embedding)
      const bool temb_staged = temb_staged_for(m_blk);
      if (p.addend != nullptr && !full_res && !temb_staged) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int mm = mrow[h] < p.M ? mrow[h] : p.M - 1;
          add_rows[h] = p.addend + static_cast<size_t>(mm / p.add_rows_per_group) * p.ld_add;
        }
      }
      mbar_wait_nocall(&vec_bar[vb], (ep >> 1) & 1);  // the service warps have staged this tile's vectors
      // LayerNorm fold: the rows' mean / rstd from their (sum, sum of squares)
      float ln_rstd[2] = {1.f, 1.f}, ln_rm[2] = {0.f, 0.f};
      if (p.stats_in) {
        const float2* s_sum = vec_lnsum(vb);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (mrow[h] >= p.M) continue;
          const float2 v = s_sum[r0 + 8 * h];
          const float sx = v.x, sxx = v.y;
          const float mean = sx * p.ln_inv_c;
          const float var = fmaxf(sxx * p.ln_inv_c - mean * mean, 0.f);
          ln_rstd[h] = rsqrtf(var + p.ln_eps);
          ln_rm[h] = ln_rstd[h] * mean;
        }
      }
      // producer side: partial row statistics [row h][column half] of this thread's columns of the tile
      float ps[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, pss[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
      if (ep > 0) mbar_wait_nocall(free_bar, (ep - 1) & 1);  // the previous tile has been read out of the staging tile
      if (full_res) mbar_wait_nocall(my_res_bar, (res_uses++) & 1);
      if (leader) {
        TL(9);
        if (tl) tl[12] = it + 1;
      }

      // The arithmetic variant (LayerNorm fold / kind of addend / row statistics) is chosen ONCE per tile and the chunk
      // loop is instantiated per variant, so the unrolled loop carries no per-element branches on them.
      if constexpr (!GEGLU) {
        auto chunks = [&](auto ln_c, auto add_c, auto st_c) {
          constexpr bool LN = decltype(ln_c)::value;
          // 0 none, 1 full residual tile, 2 staged row, 3 per-row global, 4 full residual tile + scaled result
          constexpr int ADD = decltype(add_c)::value;
          constexpr bool ST = decltype(st_c)::value;
          float res_s = 1.f;
          if constexpr (ADD == 4) res_s = *p.res_scale;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {  // 8-column group i: sub-tile i / 4, 16-byte piece i % 4
            const int col = i * 8 + cq;
            uint8_t* sub = epi_smem + (i >> 2) * C::EPI_SUB_BYTES;
            float b0 = 0.f, b1 = 0.f, sv0 = 0.f, sv1 = 0.f, tv0 = 0.f, tv1 = 0.f;
            if constexpr (LN) {
              sv0 = s_lns[col]; sv1 = s_lns[col + 1];
              tv0 = s_lnt[col]; tv1 = s_lnt[col + 1];
            } else {
              const __half2 bh = *reinterpret_cast<const __half2*>(s_bias + col);  // zeros when there is no bias
              b0 = __low2float(bh);
              b1 = __high2float(bh);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = r0 + 8 * h;
              float x0 = acc[4 * i + 2 * h], x1 = acc[4 * i + 2 * h + 1];
              if constexpr (LN) {
                x0 = x0 * ln_rstd[h] - ln_rm[h] * sv0 + tv0;
                x1 = x1 * ln_rstd[h] - ln_rm[h] * sv1 + tv1;
              } else {
                x0 += b0;
                x1 += b1;
              }
              __half2 t = __floats2half2_rn(x0, x1);
              __half2* sp = reinterpret_cast<__half2*>(sub + stage_off(r, i & 3));
              if constexpr (ADD == 4) {  // fp16(addend + fp16(t * s)): the ControlNet residual at its step's scale
                const __half2 rh = *sp;
                const __half2 ts = __floats2half2_rn(__low2float(t) * res_s, __high2float(t) * res_s);
                t = __floats2half2_rn(__low2float(rh) + __low2float(ts), __high2float(rh) + __high2float(ts));
              } else if constexpr (ADD == 1 || ADD == 2) {
                const __half2 rh = ADD == 1 ? *sp : *reinterpret_cast<const __half2*>(s_temb + col);
                t = __floats2half2_rn(__low2float(t) + __low2float(rh), __high2float(t) + __high2float(rh));
              } else if constexpr (ADD == 3) {  // tile spans several samples (tiny latents): per-row global loads
                const int n = n_blk * BN + col;
                float a0 = 0.f, a1 = 0.f;
                if (n < p.N) a0 = __half2float(add_rows[h][n]);
                if (n + 1 < p.N) a1 = __half2float(add_rows[h][n + 1]);
                t = __floats2half2_rn(__low2float(t) + a0, __high2float(t) + a1);
              }
              if constexpr (ST) {
                const float f0 = __low2float(t), f1 = __high2float(t);
                const int hc = (i < BN / 16) ? 0 : 1;
                ps[h][hc] += f0 + f1;
                pss[h][hc] += f0 * f0 + f1 * f1;
              }
              *sp = t;
            }
          }
        };
        using T = std::true_type;
        using F = std::false_type;
        const int add_mode = full_res ? 1 : (p.addend == nullptr ? 0 : (temb_staged ? 2 : 3));
        if constexpr (SCALED) {  // full residual, no fold, no statistics (host-checked)
          chunks(F{}, std::integral_constant<int, 4>{}, F{});
        } else if (p.stats_in) {  // LayerNorm-fold consumer: bias is inside t_n; no addend, no statistics (host-checked)
          chunks(T{}, std::integral_constant<int, 0>{}, F{});
        } else if (p.stats_out) {
          switch (add_mode) {
            case 0: chunks(F{}, std::integral_constant<int, 0>{}, T{}); break;
            case 1: chunks(F{}, std::integral_constant<int, 1>{}, T{}); break;
            case 2: chunks(F{}, std::integral_constant<int, 2>{}, T{}); break;
            default: chunks(F{}, std::integral_constant<int, 3>{}, T{}); break;
          }
        } else {
          switch (add_mode) {
            case 0: chunks(F{}, std::integral_constant<int, 0>{}, F{}); break;
            case 1: chunks(F{}, std::integral_constant<int, 1>{}, F{}); break;
            case 2: chunks(F{}, std::integral_constant<int, 2>{}, F{}); break;
            default: chunks(F{}, std::integral_constant<int, 3>{}, F{}); break;
          }
        }
      } else {
        // value columns [0,128), gate columns [128,256) of this tile -> 128 output columns
        auto chunks = [&](auto ln_c) {
          constexpr bool LN = decltype(ln_c)::value;
#pragma unroll
          for (int i = 0; i < BN / 16; ++i) {
            const int ia = i * 8 + cq, ig = BN / 2 + ia;
            const int ig_grp = i + BN / 16;
            uint8_t* sub = epi_smem + (i >> 2) * C::EPI_SUB_BYTES;
            float ba0 = 0.f, ba1 = 0.f, bg0 = 0.f, bg1 = 0.f;
            float sa0 = 0.f, sa1 = 0.f, ta0 = 0.f, ta1 = 0.f, sg0 = 0.f, sg1 = 0.f, tg0 = 0.f, tg1 = 0.f;
            if constexpr (LN) {
              sa0 = s_lns[ia]; sa1 = s_lns[ia + 1]; ta0 = s_lnt[ia]; ta1 = s_lnt[ia + 1];
              sg0 = s_lns[ig]; sg1 = s_lns[ig + 1]; tg0 = s_lnt[ig]; tg1 = s_lnt[ig + 1];
            } else {
              const __half2 bah = *reinterpret_cast<const __half2*>(s_bias + ia);  // zeros when there is no bias
              const __half2 bgh = *reinterpret_cast<const __half2*>(s_bias + ig);
              ba0 = __low2float(bah); ba1 = __high2float(bah);
              bg0 = __low2float(bgh); bg1 = __high2float(bgh);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float a0 = acc[4 * i + 2 * h], a1 = acc[4 * i + 2 * h + 1];
              float g0 = acc[4 * ig_grp + 2 * h], g1 = acc[4 * ig_grp + 2 * h + 1];
              if constexpr (LN) {
                a0 = a0 * ln_rstd[h] - ln_rm[h] * sa0 + ta0;
                a1 = a1 * ln_rstd[h] - ln_rm[h] * sa1 + ta1;
                g0 = g0 * ln_rstd[h] - ln_rm[h] * sg0 + tg0;
                g1 = g1 * ln_rstd[h] - ln_rm[h] * sg1 + tg1;
              } else {
                a0 += ba0; a1 += ba1;
                g0 += bg0; g1 += bg1;
              }
              const __half2 ah = __floats2half2_rn(a0, a1);
              const __half2 gh = __floats2half2_rn(g0, g1);
              const __half2 ge = __floats2half2_rn(gelu_erf_fast_f(__low2float(gh)), gelu_erf_fast_f(__high2float(gh)));
              *reinterpret_cast<__half2*>(sub + stage_off(r0 + 8 * h, i & 3)) =
                  __floats2half2_rn(__low2float(ah) * __low2float(ge), __high2float(ah) * __high2float(ge));
            }
          }
        };
        if (p.stats_in)
          chunks(std::true_type{});
        else
          chunks(std::false_type{});
      }
      fence_proxy_async_smem();  // this thread's part of the staging tile -> visible to the TMA engine
      mbar_arrive(&staged_bar[vb]);  // (and this thread is done with the tile's vectors): the store lanes take over
      if (leader) TL(13);
      if constexpr (!GEGLU) {
        if (p.stats_out) {  // quad reduction (the four lanes of a row), then one float2 per row and column half
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int hc = 0; hc < 2; ++hc) {
              ps[h][hc] += __shfl_xor_sync(0xffffffffu, ps[h][hc], 1);
              ps[h][hc] += __shfl_xor_sync(0xffffffffu, ps[h][hc], 2);
              pss[h][hc] += __shfl_xor_sync(0xffffffffu, pss[h][hc], 1);
              pss[h][hc] += __shfl_xor_sync(0xffffffffu, pss[h][hc], 2);
            }
            if ((lane & 3) == 0 && mrow[h] < p.M) {
#pragma unroll
              for (int hc = 0; hc < 2; ++hc)
                *reinterpret_cast<float2*>(p.stats_out + (static_cast<size_t>(n_blk * 2 + hc) * p.M + mrow[h]) * 2) =
                    make_float2(ps[h][hc], pss[h][hc]);
            }
          }
        }
      }
      ++ep;
    }
  }
#undef TL
}

template <int BN, bool GEGLU, bool SCALED = false>
void configure_one() {
  CFGPP_CHECK_CUDA(cudaFuncSetAttribute(gemm_kernel<BN, GEGLU, SCALED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg<BN, GEGLU>::SMEM_BYTES));
}

template <int BN, bool GEGLU, bool SCALED = false>
void launch(const GemmOp& op, cudaStream_t stream) {
  gemm_configure();
  launch_pdl(gemm_kernel<BN, GEGLU, SCALED>, dim3(op.grid), dim3(kThreads), Cfg<BN, GEGLU>::SMEM_BYTES, stream, op.p,
             op.map_a, op.map_a2, op.map_b, op.map_out, op.map_res);
}

constexpr double kSkMinSaved = 4.0;  // k-blocks of main loop the split must save per CTA
constexpr double kSkMinPiece = 0.5;  // smallest piece as a fraction of a tile's k-blocks

// Stream-K workspace: partial accumulators for up to kSkMaxCtas CTAs ([128 x 256] fp32 each) + the flag words. Launches that
// share a workspace must be stream-ordered (the flags are per CTA id), so every model handle owns one
// (StreamKScope around its plan building; a handle runs on one stream at a time) and the operator-level entry points
// fall back to one buffer per device.
thread_local float* t_sk_ws = nullptr;
thread_local unsigned* t_sk_flags = nullptr;

void streamk_buffers(float** ws, unsigned** flags) {
  if (t_sk_ws != nullptr) {  // a model handle is building its plan: its own workspace
    *ws = t_sk_ws;
    *flags = t_sk_flags;
    return;
  }
  static float* g_ws[16] = {nullptr};
  static unsigned* g_flags[16] = {nullptr};
  int dev = 0;
  CFGPP_CHECK_CUDA(cudaGetDevice(&dev));
  CFGPP_REQUIRE(dev >= 0 && dev < 16, "device index out of range");
  if (g_ws[dev] == nullptr) streamk_alloc(&g_ws[dev], &g_flags[dev]);
  *ws = g_ws[dev];
  *flags = g_flags[dev];
}

// Tile-width heuristic: time ~ rounds x (BN + 50), rounds = tiles each CTA walks. The additive term is the per-k-block
// cost that does not scale with the tile width (A-tile ingest, barrier round trip); 64-wide tiles never reach the
// tensor pipe's rate (operand fetch bound), hence their floor.
int choose_bn(int M, int N, bool geglu) {
  if (geglu) return 256;
  const int mb = (M + BM - 1) / BM;
  const int slots = std::max(1, num_sms());
  const int cand[4] = {256, 160, 128, 64};
  int best = 128;
  double best_cost = 1e30;
  for (int bn : cand) {
    if (bn == 160 && N % 160 != 0) continue;
    const int nb = (N + bn - 1) / bn;
    const long tiles = static_cast<long>(mb) * nb;
    const long rounds = (tiles + slots - 1) / slots;
    const double tile_cost = (bn < 128 ? 128 * 1.15 : bn) + 50.0;
    const double cost = rounds * tile_cost;
    if (cost < best_cost - 1e-9) {
      best_cost = cost;
      best = bn;
    }
  }
  return best;
}

void finish_op(GemmOp& op, const __half* w, int force_bn, bool force_streamk) {
  GemmParams& p = op.p;
  op.bn = force_bn ? force_bn : choose_bn(p.M, p.N, p.geglu != 0);
  CFGPP_REQUIRE(op.bn == 64 || op.bn == 128 || op.bn == 160 || op.bn == 256, "unsupported BN");
  if (p.geglu) CFGPP_REQUIRE(op.bn == 256 && p.N % 256 == 0, "GEGLU needs N % 256 == 0");
  p.num_m_blocks = (p.M + BM - 1) / BM;
  p.num_n_blocks = (p.N + op.bn - 1) / op.bn;
  // Tile walk of the linear layers: N-fastest, so the CTAs running concurrently cover few M blocks and every A tile is
  // fetched from HBM about once (large activations do not survive num_n_blocks M-fastest passes through the L2). The
  // convolutions keep the M-fastest walk.
  p.raster = p.conv ? 0 : 1;
  op.map_b = make_tmap_2d(w, p.N, p.K, p.K, op.bn);
  const int n_out = p.geglu ? p.N / 2 : p.N;
  op.map_out = make_tmap_2d_sw64(p.out, p.M, n_out, p.ldc, 16);  // one epilogue warp's [16 x 32] block
  if (p.addend != nullptr && p.add_rows_per_group <= 1) {
    CFGPP_REQUIRE(p.ld_add % 8 == 0, "residual leading dimension must be a multiple of 8");
    op.map_res = make_tmap_2d_sw64(p.addend, p.M, p.N, p.ld_add, 16);
  } else {
    op.map_res = op.map_out;
  }
  const int groups = p.num_m_blocks * p.num_n_blocks;
  const int max_ctas = num_sms();
  op.grid = groups < max_ctas ? groups : max_ctas;
  // stream-K for the remainder tiles (kernel comment "work schedule"): worth it when the left-over round would idle
  // the CTAs for at least a few k-blocks and the pieces are not slivers
  p.sk_ws = nullptr;
  p.sk_flags = nullptr;
  const int rem = groups % max_ctas;
  if (rem != 0 && max_ctas <= kSkMaxCtas) {
    // The parked partial and the fix-up cost a fixed few microseconds per launch that only long main loops amortise,
    // so the implicit-GEMM convolutions take the split and the linear layers keep the plain tile walk
    // (force_streamk, for tests, takes the split for any op whose pieces are at least 2 k-blocks deep).
    const double piece = static_cast<double>(rem) * p.num_k_blocks / max_ctas;
    const double saved = (p.num_k_blocks - piece) * op.bn / 160.0;
    // pieces at least half a tile deep (a tile then has at most three pieces, i.e. <= 2 partials to sum), unless the
    // saving is large anyway: with fewer tiles than CTAs and a long K every CTA takes a fraction of a tile
    const bool deep_enough = piece >= kSkMinPiece * p.num_k_blocks || saved >= 60.0;
    if (piece >= 2.0 && (force_streamk || (p.conv && saved >= kSkMinSaved && deep_enough))) {
      op.grid = max_ctas;  // all CTAs take part, also when there are fewer tiles than CTAs
      streamk_buffers(&p.sk_ws, &p.sk_flags);
    }
  }
}

}  // namespace

void streamk_alloc(float** ws, unsigned** flags) {
  float* w = nullptr;
  unsigned* f = nullptr;
  CFGPP_CHECK_CUDA(cudaMalloc(&w, static_cast<size_t>(kSkMaxCtas) * BM * 256 * sizeof(float)));
  try {
    CFGPP_CHECK_CUDA(cudaMalloc(&f, 2 * kSkMaxCtas * sizeof(unsigned)));
    CFGPP_CHECK_CUDA(cudaMemset(f, 0, 2 * kSkMaxCtas * sizeof(unsigned)));
    CFGPP_CHECK_CUDA(cudaDeviceSynchronize());
  } catch (...) {
    streamk_free(w, f);
    throw;
  }
  *ws = w;  // both or neither: the per-device fallback tests ws alone
  *flags = f;
}
void streamk_free(float* ws, unsigned* flags) {
  if (ws) cudaFree(ws);
  if (flags) cudaFree(flags);
}
StreamKScope::StreamKScope(float* ws, unsigned* flags) : prev_ws_(t_sk_ws), prev_flags_(t_sk_flags) {
  t_sk_ws = ws;
  t_sk_flags = flags;
}
StreamKScope::~StreamKScope() {
  t_sk_ws = prev_ws_;
  t_sk_flags = prev_flags_;
}

// opt every instantiation into its dynamic shared memory size once per process (not capturable: done eagerly)
void gemm_configure() {
  static bool done = false;
  if (done) return;
  configure_one<64, false>();
  configure_one<128, false>();
  configure_one<160, false>();
  configure_one<256, false>();
  configure_one<256, true>();
  configure_one<64, false, true>();
  configure_one<128, false, true>();
  configure_one<160, false, true>();
  configure_one<256, false, true>();
  done = true;
}

GemmOp make_linear_op(const __half* a, int lda, const __half* a2, int lda2, int k_split, const __half* w, int M,
                      int N, int K, const __half* bias, const __half* addend, int ld_add, int add_rows_per_group,
                      __half* out, int ldc, bool geglu, int force_bn, bool force_streamk) {
  GemmOp op{};
  GemmParams& p = op.p;
  CFGPP_REQUIRE(K % BK == 0, "linear K must be a multiple of 64");
  CFGPP_REQUIRE(N % 8 == 0 && ldc % 8 == 0, "N and ldc must be multiples of 8");
  p.M = M; p.N = N; p.K = K;
  p.num_k_blocks = K / BK;
  p.conv = 0; p.cpb = 1; p.H = p.W = 1; p.conv_pad = 1;
  p.k_split = a2 ? k_split : K;
  if (a2) CFGPP_REQUIRE(k_split % BK == 0 && k_split > 0 && k_split < K, "k_split must be a multiple of 64");
  p.bias = bias; p.addend = addend; p.ld_add = ld_add;
  p.add_rows_per_group = add_rows_per_group < 1 ? 1 : add_rows_per_group;
  p.out = out; p.ldc = ldc; p.geglu = geglu ? 1 : 0;
  op.map_a = make_tmap_2d(a, M, a2 ? k_split : K, lda, BM);
  op.map_a2 = a2 ? make_tmap_2d(a2, M, K - k_split, lda2, BM) : op.map_a;
  finish_op(op, w, force_bn, force_streamk);
  return op;
}

GemmOp make_conv3x3_op(const __half* x, int B, int H, int W, int Cin, const __half* w, int Cout, const __half* bias,
                       const __half* addend, int ld_add, int add_rows_per_group, __half* out, int force_bn, int stride,
                       int pad, bool force_im2col) {
  GemmOp op{};
  GemmParams& p = op.p;
  CFGPP_REQUIRE(stride == 1 || stride == 2, "conv3x3 stride must be 1 or 2");
  CFGPP_REQUIRE(pad == 1 || (pad == 0 && stride == 2), "conv3x3 pad: 1, or 0 with stride 2 (zero row / column after the image)");
  CFGPP_REQUIRE(Cin % BK == 0, "conv3x3 Cin must be a multiple of 64");
  CFGPP_REQUIRE(Cout % 8 == 0, "conv3x3 Cout must be a multiple of 8");
  CFGPP_REQUIRE(B >= 1 && H >= stride && W >= stride, "conv3x3 needs a non-empty input");
  CFGPP_REQUIRE(stride == 1 || (H % 2 == 0 && W % 2 == 0), "stride-2 conv3x3 needs even H, W");
  const int Ho = H / stride, Wo = W / stride;  // output size (pad 1, kernel 3)
  const bool im2col = force_im2col || !conv3x3_geometry_supported(Ho, Wo);
  p.M = B * Ho * Wo; p.N = Cout; p.K = 9 * Cin;
  p.num_k_blocks = 9 * (Cin / BK);
  p.conv = 1; p.cpb = Cin / BK; p.H = Ho; p.W = Wo; p.conv_stride = stride; p.conv_pad = pad;
  p.conv_im2col = im2col ? 1 : 0;
  p.k_split = p.K;
  p.bias = bias; p.addend = addend; p.ld_add = ld_add;
  p.add_rows_per_group = add_rows_per_group < 1 ? 1 : add_rows_per_group;
  p.out = out; p.ldc = Cout; p.geglu = 0;
  // the A tile of tap (kh, kw): output pixel (y, x) reads input pixel (stride * y + kh - pad, stride * x + kw - pad)
  uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
  uint32_t estr[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
  if (im2col) {
    // The walk's base pixel of output (y, x) is (stride * y - pad, stride * x - pad): the box starts at -pad and ends
    // where the last output's base lies, one pixel before the last input pixel (upper corner -1) for all three modes
    // (stride 1 pad 1: -1 .. W-2; stride 2 pad 1: -1 .. W-2, every 2nd = W/2 pixels; stride 2 pad 0: 0 .. W-2, every
    // 2nd = W/2 pixels). The taps' offsets (kw, kh) in 0..2 reach up to one pixel past the image: zero fill.
    const int lower[2] = {-pad, -pad};
    const int upper[2] = {-1, -1};
    op.map_a = make_tmap_im2col_f16(x, 4, dims, strides, lower, upper, BK, BM, estr, 128);
  } else {
    // the box spans stride * extent input pixels and the tensor map's element strides pick every stride-th one
    const int Wt = Wo < BM ? Wo : BM;
    const int Ht = (BM / Wt) < Ho ? (BM / Wt) : Ho;
    const int Nt = BM / (Wt * Ht);
    uint32_t box[4] = {64, (uint32_t)(Wt * stride), (uint32_t)(Ht * stride), (uint32_t)Nt};
    op.map_a = make_tmap_f16(x, 4, dims, strides, box, 128, estr);
  }
  op.map_a2 = op.map_a;
  finish_op(op, w, force_bn, false);
  return op;
}

GemmSchedule gemm_schedule(const GemmOp& op) {
  const GemmParams& p = op.p;
  GemmSchedule s{};
  s.bn = op.bn;
  s.grid = op.grid;
  s.tiles = p.num_m_blocks * p.num_n_blocks;
  s.streamk = p.sk_ws != nullptr ? 1 : 0;
  s.a_mode = p.conv ? (p.conv_im2col ? 2 : 1) : 0;
  s.k_blocks = p.num_k_blocks;
  s.max_pieces = 1;
  if (s.streamk && s.tiles % s.grid != 0) {
    // the kernel's "work schedule": CTA c owns units [c U / P, (c + 1) U / P) of the R * nkb remainder units
    s.sk_tiles = s.tiles % s.grid;
    const long units = static_cast<long>(s.sk_tiles) * p.num_k_blocks;
    auto u0 = [&](int c) { return units * c / s.grid; };
    for (int t = 0; t < s.sk_tiles; ++t) {
      const long b = static_cast<long>(t) * p.num_k_blocks, e = b + p.num_k_blocks;
      int pieces = 0;
      for (int c = 0; c < s.grid; ++c)
        if (u0(c + 1) > u0(c) && u0(c) < e && u0(c + 1) > b) ++pieces;
      s.max_pieces = std::max(s.max_pieces, pieces);
    }
  }
  return s;
}

void run_gemm_op(const GemmOp& op, cudaStream_t stream) {
  CFGPP_REQUIRE(!(op.p.stats_in && (op.p.addend || op.p.stats_out)),
                "a LayerNorm-fold consumer GEMM takes no addend and emits no row statistics");
  CFGPP_REQUIRE(!(op.p.stats_in && op.p.bias),
                "a LayerNorm-fold consumer GEMM takes its bias inside t_n (run_fold_ln), not as a bias vector");
  CFGPP_REQUIRE(!(op.p.geglu && (op.p.addend || op.p.stats_out)), "the GEGLU epilogue takes no addend / statistics");
  CFGPP_REQUIRE(!op.p.res_scale || (op.p.addend && op.p.add_rows_per_group <= 1 && !op.p.stats_out && !op.p.stats_in &&
                                    !op.p.geglu),
                "a scaled residual needs a full residual addend and no LayerNorm fold, statistics or GEGLU");
  if (op.p.geglu) return launch<256, true>(op, stream);
  if (op.p.res_scale) {
    switch (op.bn) {
      case 64: return launch<64, false, true>(op, stream);
      case 128: return launch<128, false, true>(op, stream);
      case 160: return launch<160, false, true>(op, stream);
      case 256: return launch<256, false, true>(op, stream);
      default: throw Error(-1, "bad BN");
    }
  }
  switch (op.bn) {
    case 64: return launch<64, false>(op, stream);
    case 128: return launch<128, false>(op, stream);
    case 160: return launch<160, false>(op, stream);
    case 256: return launch<256, false>(op, stream);
    default: throw Error(-1, "bad BN");
  }
}

}  // namespace cfgpp
