"""diffusers 0.27.1's IP-Adapter Plus restated (diffusers is not installed): `IPAdapterPlusImageProjection`, the
Perceiver "Resampler", over the image encoder's penultimate hidden states, installed through the plain adapter's
`IPAttention` processors (ip_adapter_oracle.py).

It follows diffusers, not the original IP-Adapter `Resampler`: the attention is F.scaled_dot_product_attention with
its default scale 1 / sqrt(64), where the original scales q and k each by 64^(-1/4) and rounds both to fp16 before the
product. In the dtype of the weights given (fp16 as diffusers' fp16 pipeline, or fp32 / fp64 as references), each
Linear, LayerNorm, GELU and residual add rounds once.
"""
import torch
import torch.nn.functional as F

import ip_adapter_oracle as IO


def resampler(w, h, heads, depth):
    """w: the `image_proj.*` weights; h [n, T, E] -> tokens [n, Q, D]."""
    p = "image_proj."
    x = F.linear(h, w[p + "proj_in.weight"], w[p + "proj_in.bias"])
    lat = w[p + "latents"].repeat(h.shape[0], 1, 1)
    n = h.shape[0]

    def ln(t, name):
        return F.layer_norm(t, (t.shape[-1],), w[name + ".weight"], w[name + ".bias"], 1e-5)

    def split(t):
        return t.view(n, -1, heads, t.shape[-1] // heads).transpose(1, 2)

    for i in range(depth):
        l = f"{p}layers.{i}."
        e, q_in = ln(x, l + "0.norm1"), ln(lat, l + "0.norm2")
        kv_in = torch.cat([e, q_in], dim=-2)
        k, v = F.linear(kv_in, w[l + "0.to_kv.weight"]).chunk(2, dim=-1)
        q = F.linear(q_in, w[l + "0.to_q.weight"])
        o = F.scaled_dot_product_attention(split(q), split(k), split(v))
        o = o.transpose(1, 2).reshape(n, -1, q.shape[-1])
        lat = F.linear(o, w[l + "0.to_out.weight"]) + lat
        f = F.gelu(F.linear(ln(lat, l + "1.0"), w[l + "1.1.weight"]))
        lat = F.linear(f, w[l + "1.3.weight"]) + lat
    return ln(F.linear(lat, w[p + "proj_out.weight"], w[p + "proj_out.bias"]), p + "norm_out")


def attach(model, weights, blocks, geometry):
    """Install a Plus adapter (`weights` under the native handle's keys, ip_adapter.resampler_to_unet_keys) on an
    oracle UNet. Returns the processors' state: set its tokens with `set_hidden_states`, and state["scale"]."""
    state = IO.attach(model, weights, blocks, geometry["num_queries"], None)
    state["geometry"] = geometry
    return state


def set_hidden_states(state, hidden, uncond):
    """hidden [B, T, E]: the conditional rows; uncond [1, T, E]: the encoder's hidden states of a zero image."""
    w, g = state["weights"], state["geometry"]
    dt = w["image_proj.proj_in.weight"].dtype
    h = torch.cat([uncond.to(dt).expand(hidden.shape[0], -1, -1), hidden.to(dt)])
    state["tokens"] = resampler(w, h, g["heads"], g["depth"])
