// cfgpp_b200 — wgmma GEMM / implicit-GEMM conv3x3 operator (host interface).
//
//   out[M,N] = epilogue( A[M,K] * B[N,K]^T )         fp16 in, fp32 accumulate in registers, fp16 out
//
// A is the activation in NHWC (= tokens x channels, K contiguous); B is the packed weight (N x K, K contiguous).
// Modes:
//   linear     : A through a 2D tensor map; optional second A source for K >= k_split (channel concat of
//                two tensors, used by the 1x1 shortcut conv on torch.cat([h, skip]) in up-blocks).
//   conv3x3    : stride 1, pad 1. A through a 4D tensor map (C, W, H, B); the K loop walks the 9 taps and
//                issues shifted TMA box loads whose out-of-bounds pixels are zero-filled by the hardware
//                (= the padding). Weight packed as [Cout][tap][Cin]. Two ways to fetch the A tile (the 128
//                consecutive output pixels m0 .. m0 + 127 in N·H·W order), chosen by make_conv3x3_op:
//                  tiled  : a 4-D box (64 ch, Wt, Ht, Nt) of whole row segments / rows / images — only where 128
//                           pixels form such a box (conv3x3_geometry_supported);
//                  im2col : an im2col tensor map whose 128-pixel walk wraps across row and image ends, the tap
//                           being the load's (kw, kh) offset — any geometry. Same smem tile, same k order.
// Epilogue (mirrors the rounding points of the reference's fp16 autocast graph):
//   t = fp16(acc + bias[n]);  out = addend ? fp16(float(t) + float(addend)) : t
//   addend is either a full residual [M, ld_add] or a per-sample row broadcast [M / add_rows_per_group][ld_add]
//   (the ResnetBlock2D time-embedding add).
//   Scaled residual (res_scale set, full residual only — a ControlNet zero conv adding into a UNet skip tensor):
//   out = fp16(float(addend) + float(fp16(float(t) * s))), s = *res_scale read on the device (a kernel instantiation of
//   its own: the other epilogues compile as they would without it).
//   GEGLU variant: weight rows interleaved per 256-wide tile as 128 'value' rows + 128 'gate' rows;
//   out[m, j] = fp16( fp16(a) * fp16(gelu_erf(fp16(g))) ), N_out = N / 2.
#pragma once
#include "host.h"

namespace cfgpp {

struct GemmParams {
  int M, N, K;
  int num_m_blocks, num_n_blocks, num_k_blocks;
  int conv;     // 0 linear, 1 conv3x3
  int cpb;      // conv: channel blocks (Cin / 64) per tap
  int H, W;     // conv: OUTPUT spatial size
  int conv_stride;  // conv: 1, or 2 (Downsample2D: the A tile is fetched through a tensor map with element strides 2)
  int conv_pad;     // conv: 1 (symmetric zero padding), or 0 with stride 2 (the VAE encoder's Downsample2D pads one zero
                    // row / column AFTER the image: taps at 2y + kh, out-of-image reads are the TMA's zero fill)
  int conv_im2col;  // conv: 0 = A tile through the tiled 4-D box, 1 = through the im2col map (any output geometry)
  int k_split;  // linear: first K index served by the second A map (== K when single-source)
  int raster;   // tile walk: 0 = M-fastest (tile = n * m_groups + m), 1 = N-fastest (tile = m * n_blocks + n)
  const __half* bias;
  const __half* addend;
  int ld_add;
  int add_rows_per_group;  // 1: full residual; >1: row m uses addend row (m / add_rows_per_group)
  const float* res_scale;  // full residual only: scale the tile's fp16 result by *res_scale before the add, or null
  __half* out;
  int ldc;
  int geglu;
  unsigned long long* timeline;  // debug: per-CTA timestamps (16 slots each), nullptr in production
  // ---- LayerNorm folded into the GEMM (no separate LN pass over the activations) -------------------------------
  // LN(h) W^T = rstd_m * (h (gamma (.) W)^T)_mn - rstd_m * mean_m * s_n + t_n ,  s_n = sum_k (gamma (.) W)_nk ,
  // t_n = sum_k beta_k W_nk (+ bias_n). The GEMM that PRODUCES h writes per-row partial (sum, sum of squares) of its
  // fp16 output, one slot per N block (deterministic, no atomics); the GEMM that CONSUMES LN(h) runs on h directly
  // with the folded weight and applies the row / column corrections in its epilogue.
  float* stats_out;        // producer: [2 * num_n_blocks][M] float2 (two column halves per N block), or null
  const float* stats_in;   // consumer: [ln_parts][M] float2, or null
  int ln_parts;
  float ln_inv_c, ln_eps;
  const float* ln_s;       // [N] fp32
  const float* ln_t;       // [N] fp32
  // ---- stream-K for the remainder tiles (see gemm.cu "work schedule"); null = plain data-parallel tile walk ------
  float* sk_ws;            // per CTA partial accumulator, 128 x BN fp32 in the accumulator's register order
  unsigned* sk_flags;      // [2 * 256] zero-initialised, self-resetting arrival / consumer counters
};

struct GemmOp {
  CUtensorMap map_a, map_a2, map_b, map_out, map_res;
  GemmParams p;
  int bn;
  int grid;
  // FLOP accounting (algorithmic): 2*M*N*K
  double flops() const { return 2.0 * p.M * (double)p.N * p.K; }
};

// Linear: A [M,K] with leading dim lda (elements). Optional second source a2 (cols k_split..K) with lda2.
// force_streamk (tests only): take the stream-K remainder split whenever the pieces are at least 2 k-blocks deep.
GemmOp make_linear_op(const __half* a, int lda, const __half* a2, int lda2, int k_split, const __half* w, int M,
                      int N, int K, const __half* bias, const __half* addend, int ld_add, int add_rows_per_group,
                      __half* out, int ldc, bool geglu, int force_bn = 0, bool force_streamk = false);

// Conv3x3 stride 1 pad 1 on NHWC input x [B,H,W,Cin], weight [Cout][9][Cin], out NHWC [B,H,W,Cout].
// stride 2: x is [B,H,W,Cin] with even H, W; out is [B,H/2,W/2,Cout]; pad 1 (UNet Downsample2D) or pad 0 (the
// AutoencoderKL encoder's: F.pad(x, (0, 1, 0, 1)) followed by an un-padded stride-2 convolution).
// The A tile comes through the tiled box where conv3x3_geometry_supported(output H, W) holds, through the im2col map
// otherwise; force_im2col (tests, A/B timing) takes the im2col map for every geometry.
GemmOp make_conv3x3_op(const __half* x, int B, int H, int W, int Cin, const __half* w, int Cout,
                       const __half* bias, const __half* addend, int ld_add, int add_rows_per_group, __half* out,
                       int force_bn = 0, int stride = 1, int pad = 1, bool force_im2col = false);

void run_gemm_op(const GemmOp& op, cudaStream_t stream);

// The schedule an op will run (tests: which path a launch takes on this card, without launching it).
struct GemmSchedule {
  int bn, grid, tiles;
  int streamk;     // 1: the remainder tiles are split over all CTAs (partials parked in the stream-K workspace)
  int sk_tiles;    // tiles that take the split (0 without stream-K)
  int max_pieces;  // the most pieces (CTAs) any tile is split over; 1 without stream-K
  int a_mode;      // A tile: 0 linear 2-D box, 1 conv tiled 4-D box, 2 conv im2col map
  int k_blocks;    // 64-wide k-blocks of the main loop
};
GemmSchedule gemm_schedule(const GemmOp& op);

// Stream-K workspace ownership (see gemm.cu): a model handle allocates its own buffers and wraps its plan building in a
// StreamKScope, so ops of different handles — which may run on different streams — never share flags.
void streamk_alloc(float** ws, unsigned** flags);
void streamk_free(float* ws, unsigned* flags);
class StreamKScope {
 public:
  StreamKScope(float* ws, unsigned* flags);
  ~StreamKScope();
  StreamKScope(const StreamKScope&) = delete;
  StreamKScope& operator=(const StreamKScope&) = delete;

 private:
  float* prev_ws_;
  unsigned* prev_flags_;
};

// Geometry the tiled A tile (a 4-D TMA box of 128 consecutive output pixels) can address — every other geometry takes
// the im2col A tile:
//   W > 128           : W % 128 == 0 (a tile = a 128-pixel row segment), any H;
//   W <= 128, pow2    : a tile = 128 / W whole rows: H must be a multiple of that (e.g. 96 x 128, 48 x 64, 24 x 32 —
//                       the landscape aspect buckets), or, for images smaller than a tile, H * W must divide 128
//                       (a tile = several whole images).
inline bool conv3x3_geometry_supported(int H, int W) {
  if (H < 1 || W < 1) return false;
  if (W > 128) return W % 128 == 0;
  if ((W & (W - 1)) != 0) return false;
  const int rows = 128 / W;
  return H >= rows ? (H % rows == 0) : (128 % (H * W) == 0);
}

// Latent sizes the model handles accept beyond the tiled geometry: with the im2col A tile any level runs, but the
// handles take those shapes only for latents of at least 64 x 64 (images of 512 px a side and more — the training
// resolutions of SD v1.5 / SDXL start there).
constexpr int kIm2colMinLatentSide = 64;
inline bool latent_allows_im2col(int h_lat, int w_lat) {
  return h_lat >= kIm2colMinLatentSide && w_lat >= kIm2colMinLatentSide;
}

}  // namespace cfgpp
