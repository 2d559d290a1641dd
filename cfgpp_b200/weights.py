"""UNet weights under the diffusers key scheme (SURVEY.md Appendix A.5).

The reference loads `runwayml/stable-diffusion-v1-5` / `stabilityai/stable-diffusion-xl-base-1.0` from the HF hub
(latent_diffusion.py:63, latent_sdxl.py:40) or a single-file Lightning checkpoint (latent_sdxl.py:390). Offline
there are no checkpoints, so the harness uses *seeded synthetic* weights with the real key names and shapes; a
user-supplied `*.safetensors` UNet state dict (diffusers keys) loads through the same path.
"""
from __future__ import annotations

import math
from typing import Dict, Iterator, List, Tuple

import torch

from .config import UNetConfig

Spec = Tuple[str, Tuple[int, ...], str]  # (key, shape, kind)


def _resnet(prefix: str, cin: int, cout: int, temb: int) -> Iterator[Spec]:
    yield f"{prefix}.norm1.weight", (cin,), "norm_w"
    yield f"{prefix}.norm1.bias", (cin,), "norm_b"
    yield f"{prefix}.conv1.weight", (cout, cin, 3, 3), "w"
    yield f"{prefix}.conv1.bias", (cout,), "b"
    yield f"{prefix}.time_emb_proj.weight", (cout, temb), "w"
    yield f"{prefix}.time_emb_proj.bias", (cout,), "b"
    yield f"{prefix}.norm2.weight", (cout,), "norm_w"
    yield f"{prefix}.norm2.bias", (cout,), "norm_b"
    yield f"{prefix}.conv2.weight", (cout, cout, 3, 3), "w_res"
    yield f"{prefix}.conv2.bias", (cout,), "b"
    if cin != cout:
        yield f"{prefix}.conv_shortcut.weight", (cout, cin, 1, 1), "w"
        yield f"{prefix}.conv_shortcut.bias", (cout,), "b"


def _transformer(prefix: str, c: int, layers: int, ctx: int, linear_proj: bool) -> Iterator[Spec]:
    yield f"{prefix}.norm.weight", (c,), "norm_w"
    yield f"{prefix}.norm.bias", (c,), "norm_b"
    pshape = (c, c) if linear_proj else (c, c, 1, 1)
    yield f"{prefix}.proj_in.weight", pshape, "w"
    yield f"{prefix}.proj_in.bias", (c,), "b"
    for k in range(layers):
        b = f"{prefix}.transformer_blocks.{k}"
        for n in ("norm1", "norm2", "norm3"):
            yield f"{b}.{n}.weight", (c,), "norm_w"
            yield f"{b}.{n}.bias", (c,), "norm_b"
        yield f"{b}.attn1.to_q.weight", (c, c), "w_qk"
        yield f"{b}.attn1.to_k.weight", (c, c), "w_qk"
        yield f"{b}.attn1.to_v.weight", (c, c), "w"
        yield f"{b}.attn1.to_out.0.weight", (c, c), "w_res"
        yield f"{b}.attn1.to_out.0.bias", (c,), "b"
        yield f"{b}.attn2.to_q.weight", (c, c), "w_qk"
        yield f"{b}.attn2.to_k.weight", (c, ctx), "w_qk"
        yield f"{b}.attn2.to_v.weight", (c, ctx), "w"
        yield f"{b}.attn2.to_out.0.weight", (c, c), "w_res"
        yield f"{b}.attn2.to_out.0.bias", (c,), "b"
        yield f"{b}.ff.net.0.proj.weight", (8 * c, c), "w"
        yield f"{b}.ff.net.0.proj.bias", (8 * c,), "b"
        yield f"{b}.ff.net.2.weight", (c, 4 * c), "w_res"
        yield f"{b}.ff.net.2.bias", (c,), "b"
    yield f"{prefix}.proj_out.weight", pshape, "w_res"
    yield f"{prefix}.proj_out.bias", (c,), "b"


def unet_param_specs(cfg: UNetConfig) -> List[Spec]:
    """Every parameter of UNet2DConditionModel(cfg) in diffusers naming, with its shape."""
    boc = cfg.block_out_channels
    L = len(boc)
    te = cfg.time_embed_dim
    out: List[Spec] = []
    out += [("conv_in.weight", (boc[0], cfg.in_channels, 3, 3), "w"), ("conv_in.bias", (boc[0],), "b")]
    out += [("time_embedding.linear_1.weight", (te, boc[0]), "w"), ("time_embedding.linear_1.bias", (te,), "b"),
            ("time_embedding.linear_2.weight", (te, te), "w"), ("time_embedding.linear_2.bias", (te,), "b")]
    if cfg.addition_embed_type == "text_time":
        ain = cfg.projection_class_embeddings_input_dim
        out += [("add_embedding.linear_1.weight", (te, ain), "w"), ("add_embedding.linear_1.bias", (te,), "b"),
                ("add_embedding.linear_2.weight", (te, te), "w"), ("add_embedding.linear_2.bias", (te,), "b")]
    ch = boc[0]
    for i in range(L):
        cin, ch = ch, boc[i]
        for j in range(cfg.layers_per_block):
            out += list(_resnet(f"down_blocks.{i}.resnets.{j}", cin if j == 0 else ch, ch, te))
            if cfg.down_block_types[i] == "CrossAttnDownBlock2D":
                out += list(_transformer(f"down_blocks.{i}.attentions.{j}", ch, cfg.transformer_layers_per_block[i],
                                         cfg.cross_attention_dim, cfg.use_linear_projection))
        if i != L - 1:
            out += [(f"down_blocks.{i}.downsamplers.0.conv.weight", (ch, ch, 3, 3), "w"),
                    (f"down_blocks.{i}.downsamplers.0.conv.bias", (ch,), "b")]
    cm = boc[-1]
    out += list(_resnet("mid_block.resnets.0", cm, cm, te))
    out += list(_transformer("mid_block.attentions.0", cm, cfg.transformer_layers_per_block[-1],
                             cfg.cross_attention_dim, cfg.use_linear_projection))
    out += list(_resnet("mid_block.resnets.1", cm, cm, te))
    rev = list(reversed(boc))
    ch = rev[0]
    for i in range(L):
        prev, ch = ch, rev[i]
        cin = rev[min(i + 1, L - 1)]
        n = cfg.layers_per_block + 1
        for j in range(n):
            skip = cin if j == n - 1 else ch
            rin = prev if j == 0 else ch
            out += list(_resnet(f"up_blocks.{i}.resnets.{j}", rin + skip, ch, te))
            if cfg.up_block_types[i] == "CrossAttnUpBlock2D":
                out += list(_transformer(f"up_blocks.{i}.attentions.{j}", ch,
                                         cfg.transformer_layers_per_block[L - 1 - i], cfg.cross_attention_dim,
                                         cfg.use_linear_projection))
        if i != L - 1:
            out += [(f"up_blocks.{i}.upsamplers.0.conv.weight", (ch, ch, 3, 3), "w"),
                    (f"up_blocks.{i}.upsamplers.0.conv.bias", (ch,), "b")]
    out += [("conv_norm_out.weight", (boc[0],), "norm_w"), ("conv_norm_out.bias", (boc[0],), "norm_b"),
            ("conv_out.weight", (cfg.out_channels, boc[0], 3, 3), "w_out"), ("conv_out.bias", (cfg.out_channels,), "b")]
    return out


def num_params(cfg: UNetConfig) -> int:
    return sum(math.prod(s) for _, s, _ in unet_param_specs(cfg))


def synthetic_state_dict(cfg: UNetConfig, seed: int = 1234, device="cpu", dtype=torch.float16) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights with activation-preserving scales (unit-gain matrices, attention logits of O(1),
    damped residual branches) so that every kernel sees realistic dynamic range. Values are generated in fp32 on
    `device` and stored as `dtype`; the fp16 values ARE the model (the fp32 oracle upcasts the same fp16 numbers)."""
    return synthetic_from_specs(unet_param_specs(cfg), seed, device, dtype)


def synthetic_from_specs(specs: List[Spec], seed: int = 1234, device="cpu",
                         dtype=torch.float16) -> Dict[str, torch.Tensor]:
    """The seeded weights of synthetic_state_dict for any list of (key, shape, kind) specs, drawn in list order."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for key, shape, kind in specs:
        if kind == "norm_w":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        elif kind in ("norm_b", "b"):
            t = 0.05 * torch.randn(shape, generator=g, device=device)
        else:
            fan_in = math.prod(shape[1:])
            gain = {"w": 1.0, "w_qk": 1.2, "w_res": 0.4, "w_out": 1.0}[kind]
            t = torch.randn(shape, generator=g, device=device) * (gain / math.sqrt(fan_in))
        sd[key] = t.to(dtype)
    return sd


def load_safetensors_state_dict(path: str, device="cpu", dtype=torch.float16) -> Dict[str, torch.Tensor]:
    """A diffusers-format UNet `*.safetensors` (the file `ckpt/` is meant to hold, reference README.md:67)."""
    from safetensors.torch import load_file
    return {k: v.to(device=device, dtype=dtype) for k, v in load_file(path).items()}
