// cfgpp_b200 — fused scaled-dot-product attention (no mask, no dropout) on the sm_90a tensor cores.
//   out[b, i, h*P + :] = softmax(q_i k^T / sqrt(d)) v           (AttnProcessor2_0 / F.scaled_dot_product_attention)
// d = real head dim (SDXL: 64; SD v1.5: 40 / 80 / 160), P = d rounded up to a multiple of 64: the projections that
// feed this kernel emit each head zero-padded to P columns (and to_out ignores the padded columns), so every tile is
// made of whole 128-byte swizzle atoms. q / k / v are strided views into token-major activation buffers
// ([B*N, ld] fp16, head h at column h*P): the fused QKV / KV GEMM outputs are consumed in place; the output is written
// token-major [B*Nq, ldo] ready for the to_out GEMM.
#pragma once
#include "host.h"

namespace cfgpp {

struct AttnParams {
  int B, H, Nq, Nkv;
  int ldo;
  __half* out;
  float scale_log2e;  // (1/sqrt(d)) * log2(e)
};

struct AttnOp {
  CUtensorMap map_q, map_k, map_v;
  AttnParams p;
  int hd_pad;
  int head_dim;
  double flops() const { return 4.0 * p.B * p.H * (double)p.Nq * p.Nkv * head_dim; }  // algorithmic (unpadded)
};

int attn_padded_head_dim(int head_dim);
AttnOp make_attn_op(const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, __half* out,
                    int ldo, int B, int H, int Nq, int Nkv, int head_dim = 64);
void run_attn_op(const AttnOp& op, cudaStream_t stream);

}  // namespace cfgpp
