"""IP-Adapter (Ye et al. 2023, `h94/IP-Adapter`): a reference image as a prompt, through decoupled cross-attention.

An adapter is an image projection (diffusers `ImageProjection`: Linear(E -> n_tokens * D), then LayerNorm(D) per
token) and one pair of K / V projections `to_k_ip` / `to_v_ip` [C, D] per cross-attention of the UNet. Every `attn2`
then attends to the text tokens and, with a softmax of its own, to the n_tokens image tokens, and adds the second
result at a scale s (see `cfgpp_ip_adapter_attach` in include/cfgpp_b200.h for the arithmetic).

The original checkpoints number the K / V pairs `ip_adapter.{i}` by processor index: every `attn1` and `attn2` of the
UNet counted in diffusers' `attn_processors` order, which is down blocks, up blocks, then the mid block (the order in
which `UNet2DConditionModel` registers them), so `attn2` sits at the odd indices. `processor_blocks` is the one place
that mapping is made; the native handle takes the weights under the UNet-side keys it maps to.
"""
from __future__ import annotations

import zlib
from pathlib import Path
from typing import Dict, List, Optional

import torch

from .config import UNetConfig

KV_SUFFIX = {"to_k_ip": ".attn2.processor.to_k_ip.0.weight", "to_v_ip": ".attn2.processor.to_v_ip.0.weight"}
MAX_TOKENS = 64


def attn2_blocks(cfg: UNetConfig) -> List[str]:
    """The transformer blocks of the UNet in diffusers' `attn_processors` order: down blocks, up blocks, mid block."""
    L, lpb = len(cfg.block_out_channels), cfg.layers_per_block
    tl = cfg.transformer_layers_per_block
    out = []
    for i in range(L):
        if cfg.down_block_types[i].startswith("CrossAttn"):
            for j in range(lpb):
                out += [f"down_blocks.{i}.attentions.{j}.transformer_blocks.{k}" for k in range(tl[i])]
    for i in range(L):
        if cfg.up_block_types[i].startswith("CrossAttn"):
            for j in range(lpb + 1):
                out += [f"up_blocks.{i}.attentions.{j}.transformer_blocks.{k}" for k in range(tl[L - 1 - i])]
    out += [f"mid_block.attentions.0.transformer_blocks.{k}" for k in range(tl[L - 1])]
    return out


def processor_blocks(cfg: UNetConfig) -> Dict[int, str]:
    """{processor index of an attn2: its transformer block}: the odd indices 1, 3, …, 2·n − 1."""
    return {2 * n + 1: b for n, b in enumerate(attn2_blocks(cfg))}


def block_channels(cfg: UNetConfig) -> Dict[str, int]:
    """The width C of every transformer block (the rows of its to_k_ip / to_v_ip)."""
    L, ch = len(cfg.block_out_channels), cfg.block_out_channels
    out = {}
    for b in attn2_blocks(cfg):
        kind, i = b.split(".")[:2]
        out[b] = ch[int(i)] if kind == "down_blocks" else ch[L - 1 - int(i)] if kind == "up_blocks" else ch[L - 1]
    return out


def synthetic_ip_adapter(cfg: UNetConfig, embed_dim: int, n_tokens: int = 4, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded fp32 weights under the original checkpoint's flat keys (`image_proj.*`, `ip_adapter.{i}.*`), shaped for
    the base UNet `cfg`; each matrix has std 1 / sqrt(fan_in), the norm gamma ≈ 1."""
    g = torch.Generator().manual_seed(seed)
    D = cfg.cross_attention_dim

    def rn(*s):
        return torch.randn(*s, generator=g) / s[-1] ** 0.5

    sd = {"image_proj.proj.weight": rn(n_tokens * D, embed_dim),
          "image_proj.proj.bias": 0.1 * torch.randn(n_tokens * D, generator=g),
          "image_proj.norm.weight": 1 + 0.1 * torch.randn(D, generator=g),
          "image_proj.norm.bias": 0.1 * torch.randn(D, generator=g)}
    C = block_channels(cfg)
    for i, b in processor_blocks(cfg).items():
        sd[f"ip_adapter.{i}.to_k_ip.weight"] = rn(C[b], D)
        sd[f"ip_adapter.{i}.to_v_ip.weight"] = rn(C[b], D)
    return sd


def read_ip_adapter_file(path) -> Dict[str, torch.Tensor]:
    """The flat state dict of an original checkpoint: a `.bin` holding {"image_proj": {...}, "ip_adapter": {...}}, or
    a `.safetensors` with `image_proj.*` / `ip_adapter.*` keys."""
    path = Path(path)
    if path.suffix == ".safetensors":
        from safetensors.torch import load_file
        return dict(load_file(str(path)))
    sd = torch.load(str(path), map_location="cpu", weights_only=True)
    if not (isinstance(sd, dict) and set(sd) == {"image_proj", "ip_adapter"}):
        raise ValueError(f"{path}: expected a dict with the keys 'image_proj' and 'ip_adapter'")
    return {f"{top}.{k}": v for top in ("image_proj", "ip_adapter") for k, v in sd[top].items()}


def to_unet_keys(sd: Dict[str, torch.Tensor], cfg: UNetConfig):
    """Validate a flat original state dict against the base UNet and map it to the native handle's keys.
    Returns (weights, n_tokens, embed_dim). ValueError names the offending key: an unknown key, a projection other
    than the plain Linear + LayerNorm one (Resampler, MLP), a missing attn2 index or a shape that does not fit."""
    D = cfg.cross_attention_dim
    blocks, C = processor_blocks(cfg), block_channels(cfg)
    proj = {"image_proj.proj.weight", "image_proj.proj.bias", "image_proj.norm.weight", "image_proj.norm.bias"}
    out = {}
    for key, t in sd.items():
        if key.startswith("image_proj."):
            if key not in proj:
                raise ValueError(f"{key}: unsupported image projection (only IP-Adapter's Linear + LayerNorm "
                                 "ImageProjection; the Plus Resampler and the Full-Face MLP are not implemented)")
            out[key] = t
            continue
        parts = key.split(".")
        if len(parts) != 4 or parts[0] != "ip_adapter" or not parts[1].isdigit() or parts[2] not in KV_SUFFIX \
                or parts[3] != "weight":
            raise ValueError(f"{key}: not an IP-Adapter weight")
        i = int(parts[1])
        if i not in blocks:
            raise ValueError(f"{key}: processor index {i} is not a cross-attention of this UNet "
                             f"(attn2 sits at the odd indices 1..{2 * len(blocks) - 1})")
        b = blocks[i]
        if tuple(t.shape) != (C[b], D):
            raise ValueError(f"{key}: shape {tuple(t.shape)}, the UNet's {b}.attn2 needs {(C[b], D)}")
        out[b + KV_SUFFIX[parts[2]]] = t
    missing = sorted(proj - set(out))
    if missing:
        raise ValueError(f"{missing[0]}: missing")
    for i, b in blocks.items():
        for name, suffix in KV_SUFFIX.items():
            if b + suffix not in out:
                raise ValueError(f"ip_adapter.{i}.{name}.weight: missing (attn2 of {b})")
    w = out["image_proj.proj.weight"]
    if w.dim() != 2 or w.shape[0] % D != 0 or not 1 <= w.shape[0] // D <= MAX_TOKENS:
        raise ValueError(f"image_proj.proj.weight: shape {tuple(w.shape)} is not [n_tokens * {D}, E], "
                         f"n_tokens 1..{MAX_TOKENS}")
    n_tokens, embed_dim = w.shape[0] // D, w.shape[1]
    if embed_dim % 8:
        raise ValueError(f"image_proj.proj.weight: image embedding width {embed_dim} is not a multiple of 8")
    for key, shape in (("image_proj.proj.bias", (n_tokens * D,)), ("image_proj.norm.weight", (D,)),
                       ("image_proj.norm.bias", (D,))):
        if tuple(out[key].shape) != shape:
            raise ValueError(f"{key}: shape {tuple(out[key].shape)}, expected {shape}")
    return out, n_tokens, embed_dim


def default_encoder_config(base_cfg: UNetConfig):
    """The image encoder a base UNet's adapters were trained with: ViT-bigG/14 for SDXL, ViT-H/14 for SD v1.5; the tiny
    test UNets get the tiny test tower."""
    from . import vision_encoder as V
    if base_cfg.name.startswith("tiny"):
        return V.tiny_vision_config()
    return V.vit_bigg_config() if base_cfg.addition_embed_type == "text_time" else V.vit_h_config()


class IPAdapter:
    """One IP-Adapter for a base UNet, with its CLIP vision tower. `path_or_key` is a `.bin` / `.safetensors`
    checkpoint (a path with one of those suffixes that does not exist is an error), or any other key, which gets
    seeded synthetic weights. `image_encoder` is an image-encoder directory (`config.json` + `model.safetensors`), or
    None for a seeded synthetic tower of the base UNet's kind (`default_encoder_config`). The adapter's image embedding
    width must equal the tower's projection_dim."""

    def __init__(self, path_or_key: str, device, base_cfg: UNetConfig, image_encoder: Optional[str] = None,
                 n_tokens: int = 4):
        from . import vision_encoder as V
        self.device = torch.device(device)
        if image_encoder is not None:
            self.encoder_cfg, enc_sd = V.load_encoder_dir(image_encoder)
        else:
            self.encoder_cfg = default_encoder_config(base_cfg)
            enc_sd = V.synthetic_state_dict(self.encoder_cfg, seed=zlib.crc32(f"{path_or_key}:encoder".encode())
                                            & 0x7FFFFFFF, device=self.device if self.device.type == "cuda" else "cpu")
        p = Path(path_or_key)
        if p.suffix in (".bin", ".safetensors"):
            if not p.is_file():
                raise FileNotFoundError(f"IP-Adapter checkpoint {path_or_key} does not exist")
            sd = read_ip_adapter_file(p)
        else:
            sd = synthetic_ip_adapter(base_cfg, self.encoder_cfg.projection_dim, n_tokens,
                                      seed=zlib.crc32(path_or_key.encode()) & 0x7FFFFFFF)
        if base_cfg.prediction_type != "epsilon" or base_cfg.name.split("_")[-1] not in ("sd15", "sdxl"):
            raise ValueError(f"IP-Adapter conditions SD v1.5 and SDXL UNets, not {base_cfg.name}")
        self.key, self.base_cfg = path_or_key, base_cfg
        self.state_dict = sd
        self.weights, self.n_tokens, self.embed_dim = to_unet_keys(sd, base_cfg)
        if self.embed_dim != self.encoder_cfg.projection_dim:
            raise ValueError(f"image_proj.proj.weight: the adapter takes {self.embed_dim}-wide image embeddings, the "
                             f"image encoder gives {self.encoder_cfg.projection_dim}")
        self._enc_sd = enc_sd
        self._encoder = None

    @property
    def encoder(self):
        """The native vision tower (built on first use)."""
        if self._encoder is None:
            from . import vision_encoder as V
            self._encoder = V.NativeCLIPVisionEncoder(self.encoder_cfg, self._enc_sd, self.device)
            self._enc_sd = None
        return self._encoder

    def image_embeds(self, images, batch: int) -> torch.Tensor:
        """`images`: one image (PIL, uint8 (H, W, 3) array, or a (3, H, W) / (1, 3, H, W) tensor in [0, 1]) for every
        prompt, or a sequence of `batch` of them -> image_embeds (batch, E) fp16 on the device."""
        from . import vision_encoder as V
        if isinstance(images, torch.Tensor):
            t = images.detach().float().cpu()
            t = t.unsqueeze(0) if t.dim() == 3 else t
            images = [(x.clamp(0, 1).permute(1, 2, 0) * 255).round().to(torch.uint8).numpy() for x in t]
        elif not isinstance(images, (list, tuple)):
            images = [images]
        if len(images) not in (1, batch):
            raise ValueError(f"ip_adapter_image: {len(images)} images for {batch} prompts (give one, or one per prompt)")
        e = self.encoder.encode(V.preprocess(images, self.encoder_cfg.image_size))
        return e.expand(batch, -1).contiguous() if e.shape[0] == 1 else e

    def close(self):
        if self._encoder is not None:
            self._encoder.close()
            self._encoder = None
