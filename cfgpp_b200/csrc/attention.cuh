// cfgpp_b200 — fused scaled-dot-product attention (no mask, no dropout) on the sm_90a tensor cores.
//   out[b, i, h*P + :] = softmax(q_i k^T / sqrt(d)) v           (AttnProcessor2_0 / F.scaled_dot_product_attention)
// d = real head dim (SDXL: 64; SD v1.5: 40 / 80 / 160), P = d rounded up to a multiple of 64: the projections that
// feed this kernel emit each head zero-padded to P columns (and to_out ignores the padded columns), so every tile is
// made of whole 128-byte swizzle atoms. q / k / v are strided views into token-major activation buffers
// ([B*N, ld] fp16, head h at column h*P): the fused QKV / KV GEMM outputs are consumed in place; the output is written
// token-major [B*Nq, ldo] ready for the to_out GEMM.
//
// Decoupled cross-attention (IP-Adapter, make_attn_ip_op): the query also attends to Nkv2 <= 64 image tokens k2 / v2
// (same head layout) under a softmax of its own, and
//   out[b, i, h*P + :] = fp16( O1 / l1 + s * O2 / l2 ),   O / l = the unnormalised PV and the sum of each segment,
// s = *ip_scale, an fp32 device word read by every launch (a captured graph follows it). The text half is the plain
// kernel's arithmetic; the sum is formed in fp32 and rounded once. diffusers (IPAdapterAttnProcessor2_0) rounds each
// term first: fp16(fp16(O_txt) + fp16(s * fp16(O_ip))); the two differ by at most an ulp or so of each term. At s = 0
// the output is the plain kernel's, bit for bit (head dims 128 / 192 skip the image tile; head dim 64 computes it and
// drops it by a select).
#pragma once
#include "host.h"

namespace cfgpp {

struct AttnParams {
  int B, H, Nq, Nkv;
  int ldo;
  __half* out;
  float scale_log2e;  // (1/sqrt(d)) * log2(e)
  int Nkv2;                // image tokens (decoupled cross-attention only)
  const float* ip_scale;   // device word s; null: plain attention
};

struct AttnOp {
  CUtensorMap map_q, map_k, map_v;
  CUtensorMap map_k2, map_v2;  // image tokens (decoupled cross-attention only)
  AttnParams p;
  int hd_pad;
  int head_dim;
  double flops() const {  // algorithmic (unpadded)
    return 4.0 * p.B * p.H * (double)p.Nq * (p.Nkv + (p.ip_scale ? p.Nkv2 : 0)) * head_dim;
  }
};

int attn_padded_head_dim(int head_dim);
AttnOp make_attn_op(const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, __half* out,
                    int ldo, int B, int H, int Nq, int Nkv, int head_dim = 64);
// k2 / v2 [B*Nkv2, ld] in the layout of k / v; ip_scale: device pointer to s (fp32)
AttnOp make_attn_ip_op(const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, const __half* k2,
                       int ldk2, const __half* v2, int ldv2, int Nkv2, const float* ip_scale, __half* out, int ldo,
                       int B, int H, int Nq, int Nkv, int head_dim);
void run_attn_op(const AttnOp& op, cudaStream_t stream);

}  // namespace cfgpp
