"""diffusers' IP-Adapter restated on the oracle UNet (diffusers is not installed): `ImageProjection` (Linear, reshape to
tokens, LayerNorm) and `IPAdapterAttnProcessor2_0` in place of every attn2. The processor computes the text attention
as oracle/unet.py's Attention does, the image attention with the same query, adds the second at the scale, then runs
to_out: under fp16 autocast each term and the sum are rounded to fp16, as diffusers' fp16 pipeline does."""
import torch
import torch.nn.functional as F
from torch import nn


def image_tokens(weights, embeds, n_tokens, D):
    """ImageProjection of embeds [rows, E] -> [rows, n_tokens, D]."""
    x = F.linear(embeds, weights["image_proj.proj.weight"], weights["image_proj.proj.bias"])
    x = x.reshape(embeds.shape[0], n_tokens, D)
    return F.layer_norm(x, (D,), weights["image_proj.norm.weight"], weights["image_proj.norm.bias"], 1e-5)


class IPAttention(nn.Module):
    """attn2 of one transformer block with the decoupled image attention; `state` holds the tokens and the scale."""

    def __init__(self, attn, wk, wv, state):
        super().__init__()
        self.attn, self.state = attn, state
        self.register_buffer("wk", wk)
        self.register_buffer("wv", wv)

    def forward(self, hidden_states, encoder_hidden_states=None):
        a = self.attn
        b, heads = hidden_states.shape[0], a.heads

        def split(t):
            return t.view(b, -1, heads, t.shape[-1] // heads).transpose(1, 2)

        q = split(a.to_q(hidden_states))
        o = F.scaled_dot_product_attention(q, split(a.to_k(encoder_hidden_states)),
                                           split(a.to_v(encoder_hidden_states)))
        tok = self.state["tokens"]
        o_ip = F.scaled_dot_product_attention(q, split(F.linear(tok, self.wk)), split(F.linear(tok, self.wv)))
        o = o + self.state["scale"] * o_ip
        o = o.transpose(1, 2).reshape(b, -1, heads * q.shape[-1]).to(q.dtype)
        return a.to_out[0](o)


def attach(model, weights, blocks, n_tokens, D):
    """Install the adapter (`weights` under the native handle's keys, cfgpp_b200.ip_adapter.to_unet_keys) on an oracle
    UNet. Returns the state dict the processors read: set state["tokens"] with `set_embeds` and state["scale"]."""
    p = next(model.parameters())
    w = {k: v.to(device=p.device, dtype=p.dtype) for k, v in weights.items()}
    state = {"scale": 1.0, "tokens": None, "weights": w, "n_tokens": n_tokens, "D": D}
    for b in blocks:
        tb = model.get_submodule(b)
        tb.attn2 = IPAttention(tb.attn2, w[b + ".attn2.processor.to_k_ip.0.weight"],
                               w[b + ".attn2.processor.to_v_ip.0.weight"], state)
    return state


def set_embeds(state, embeds):
    """embeds [B, E] of the conditional rows; the unconditional rows get zeros (diffusers' negative image embeds)."""
    e = embeds.to(state["weights"]["image_proj.proj.weight"].dtype)
    state["tokens"] = image_tokens(state["weights"], torch.cat([torch.zeros_like(e), e]), state["n_tokens"], state["D"])
