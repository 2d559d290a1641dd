"""IP-Adapter (Ye et al. 2023, `h94/IP-Adapter`): a reference image as a prompt, through decoupled cross-attention.

An adapter is an image projection (diffusers `ImageProjection`: Linear(E -> n_tokens * D), then LayerNorm(D) per
token) and one pair of K / V projections `to_k_ip` / `to_v_ip` [C, D] per cross-attention of the UNet. Every `attn2`
then attends to the text tokens and, with a softmax of its own, to the n_tokens image tokens, and adds the second
result at a scale s (see `cfgpp_ip_adapter_attach` in include/cfgpp_b200.h for the arithmetic).

The original checkpoints number the K / V pairs `ip_adapter.{i}` by processor index: every `attn1` and `attn2` of the
UNet counted in diffusers' `attn_processors` order, which is down blocks, up blocks, then the mid block (the order in
which `UNet2DConditionModel` registers them), so `attn2` sits at the odd indices. `processor_blocks` is the one place
that mapping is made; the native handle takes the weights under the UNet-side keys it maps to.

IP-Adapter Plus (`ip-adapter-plus*`) replaces the image projection by a Perceiver "Resampler" (diffusers
`IPAdapterPlusImageProjection`) that reads the image encoder's penultimate hidden states [n, T, E] and returns Q image
tokens; its unconditional rows are the encoder's hidden states of an all-zero preprocessed image, not zeros. A state
dict is a Resampler iff it has `image_proj.latents` and no `image_proj.proj.weight` (`is_resampler`);
`resampler_to_unet_keys` is its census.
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


def _kv_unet_key(key: str, t: torch.Tensor, cfg: UNetConfig, blocks: Dict[int, str], C: Dict[str, int]) -> str:
    """The native handle's key of the original K / V weight `key` (`ip_adapter.{i}.to_{k,v}_ip.weight`)."""
    parts = key.split(".")
    if len(parts) != 4 or parts[0] != "ip_adapter" or not parts[1].isdigit() or parts[2] not in KV_SUFFIX \
            or parts[3] != "weight":
        raise ValueError(f"{key}: not an IP-Adapter weight")
    i = int(parts[1])
    if i not in blocks:
        raise ValueError(f"{key}: processor index {i} is not a cross-attention of this UNet "
                         f"(attn2 sits at the odd indices 1..{2 * len(blocks) - 1})")
    b = blocks[i]
    if tuple(t.shape) != (C[b], cfg.cross_attention_dim):
        raise ValueError(f"{key}: shape {tuple(t.shape)}, the UNet's {b}.attn2 needs {(C[b], cfg.cross_attention_dim)}")
    return b + KV_SUFFIX[parts[2]]


def _require_every_kv(out: Dict[str, torch.Tensor], blocks: Dict[int, str]) -> None:
    for i, b in blocks.items():
        for name, suffix in KV_SUFFIX.items():
            if b + suffix not in out:
                raise ValueError(f"ip_adapter.{i}.{name}.weight: missing (attn2 of {b})")


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
        out[_kv_unet_key(key, t, cfg, blocks, C)] = t
    missing = sorted(proj - set(out))
    if missing:
        raise ValueError(f"{missing[0]}: missing")
    _require_every_kv(out, blocks)
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


RESAMPLER_TOP = ("latents", "proj_in.weight", "proj_in.bias", "proj_out.weight", "proj_out.bias", "norm_out.weight",
                 "norm_out.bias")
RESAMPLER_LAYER = ("0.norm1.weight", "0.norm1.bias", "0.norm2.weight", "0.norm2.bias", "0.to_q.weight", "0.to_kv.weight",
                   "0.to_out.weight", "1.0.weight", "1.0.bias", "1.1.weight", "1.3.weight")
HEAD_DIM = 64


def is_resampler(sd: Dict[str, torch.Tensor]) -> bool:
    """An IP-Adapter Plus state dict: `image_proj.latents` present, `image_proj.proj.weight` absent."""
    return "image_proj.latents" in sd and "image_proj.proj.weight" not in sd


def resampler_shapes(g: dict, D: int) -> Dict[str, tuple]:
    """{image_proj.* key: shape} of a Resampler of geometry g (num_queries, embed_dim, dim, heads, depth, ff_mult)
    producing D-wide tokens."""
    Q, E, dim, depth = g["num_queries"], g["embed_dim"], g["dim"], g["depth"]
    inner, F = HEAD_DIM * g["heads"], g["ff_mult"] * g["dim"]
    out = {"latents": (1, Q, dim), "proj_in.weight": (dim, E), "proj_in.bias": (dim,), "proj_out.weight": (D, dim),
           "proj_out.bias": (D,), "norm_out.weight": (D,), "norm_out.bias": (D,)}
    per = {"0.norm1.weight": (dim,), "0.norm1.bias": (dim,), "0.norm2.weight": (dim,), "0.norm2.bias": (dim,),
           "0.to_q.weight": (inner, dim), "0.to_kv.weight": (2 * inner, dim), "0.to_out.weight": (dim, inner),
           "1.0.weight": (dim,), "1.0.bias": (dim,), "1.1.weight": (F, dim), "1.3.weight": (dim, F)}
    for i in range(depth):
        out.update({f"layers.{i}.{k}": v for k, v in per.items()})
    return {"image_proj." + k: v for k, v in out.items()}


def resampler_to_unet_keys(sd: Dict[str, torch.Tensor], cfg: UNetConfig):
    """The census of an IP-Adapter Plus state dict: validate it against the base UNet and map it to the native
    handle's keys (the `image_proj.*` keys stay as they are). Returns (weights, geometry), geometry = {num_queries,
    embed_dim, dim, heads, depth, ff_mult} inferred as diffusers does (heads = rows(to_q) / 64). ValueError names the
    offending key: one that is not part of the Resampler (the Full-Face MLP, `pos_emb`,
    `to_latents_from_mean_pooled_seq`), a missing one, or a shape that does not fit."""
    blocks, C = processor_blocks(cfg), block_channels(cfg)
    out, layers = {}, set()
    for key, t in sd.items():
        if not key.startswith("image_proj."):
            out[_kv_unet_key(key, t, cfg, blocks, C)] = t
            continue
        k = key[len("image_proj."):]
        parts = k.split(".")
        if k in RESAMPLER_TOP:
            pass
        elif len(parts) > 2 and parts[0] == "layers" and parts[1].isdigit() and ".".join(parts[2:]) in RESAMPLER_LAYER:
            layers.add(int(parts[1]))
        else:
            raise ValueError(f"{key}: not a weight of the IP-Adapter Plus Resampler (its position embedding, mean-pooled "
                             "latents and the Full-Face MLP projection are not implemented)")
        out[key] = t
    for k in RESAMPLER_TOP:
        if "image_proj." + k not in out:
            raise ValueError(f"image_proj.{k}: missing")
    depth = max(layers) + 1 if layers else 0
    if depth == 0:
        raise ValueError("image_proj.layers.0.0.to_q.weight: missing (a Resampler has at least one layer)")
    for i in range(depth):
        for n in RESAMPLER_LAYER:
            if f"image_proj.layers.{i}.{n}" not in out:
                raise ValueError(f"image_proj.layers.{i}.{n}: missing")
    lat, pin = out["image_proj.latents"], out["image_proj.proj_in.weight"]
    wq, w1 = out["image_proj.layers.0.0.to_q.weight"], out["image_proj.layers.0.1.1.weight"]
    if lat.dim() != 3 or lat.shape[0] != 1 or not 1 <= lat.shape[1] <= MAX_TOKENS or lat.shape[2] % 64:
        raise ValueError(f"image_proj.latents: shape {tuple(lat.shape)} is not [1, Q, dim] with Q 1..{MAX_TOKENS} "
                         "and dim a multiple of 64")
    dim = lat.shape[2]
    if pin.dim() != 2 or pin.shape[1] % 64:
        raise ValueError(f"image_proj.proj_in.weight: shape {tuple(pin.shape)} is not [dim, E] with E a multiple of 64")
    if wq.dim() != 2 or wq.shape[0] % HEAD_DIM or wq.shape[0] == 0:
        raise ValueError(f"image_proj.layers.0.0.to_q.weight: shape {tuple(wq.shape)}: its rows are not a whole number "
                         f"of {HEAD_DIM}-wide heads")
    if w1.dim() != 2 or w1.shape[0] % dim or w1.shape[0] == 0:
        raise ValueError(f"image_proj.layers.0.1.1.weight: shape {tuple(w1.shape)}: its rows are not a multiple of "
                         f"dim {dim}")
    g = {"num_queries": lat.shape[1], "embed_dim": pin.shape[1], "dim": dim, "heads": wq.shape[0] // HEAD_DIM,
         "depth": depth, "ff_mult": w1.shape[0] // dim}
    for key, shape in resampler_shapes(g, cfg.cross_attention_dim).items():
        if tuple(out[key].shape) != shape:
            raise ValueError(f"{key}: shape {tuple(out[key].shape)}, expected {shape}")
    _require_every_kv(out, blocks)
    return out, g


def plus_geometry(cfg: UNetConfig, embed_dim: int) -> dict:
    """The released Plus adapters' Resampler for a base UNet (SD v1.5: dim 768, 12 heads; SDXL: dim 1280, 20 heads;
    16 queries, 4 layers, ff_mult 4); the tiny test UNets get a 2-layer, 2-head, 128-wide one."""
    dim, heads, depth = ((128, 2, 2) if cfg.name.startswith("tiny") else
                         (1280, 20, 4) if cfg.addition_embed_type == "text_time" else (768, 12, 4))
    return {"num_queries": 16, "embed_dim": embed_dim, "dim": dim, "heads": heads, "depth": depth, "ff_mult": 4}


def synthetic_ip_adapter_plus(cfg: UNetConfig, geometry: dict, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded fp32 IP-Adapter Plus weights under the original checkpoint's flat keys; each matrix has std
    1 / sqrt(fan_in), the latents std 1 / sqrt(dim) (as diffusers initialises them), the norm gammas ≈ 1."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key, shape in resampler_shapes(geometry, cfg.cross_attention_dim).items():
        if key.endswith("norm1.weight") or key.endswith("norm2.weight") or key.endswith("1.0.weight") \
                or key == "image_proj.norm_out.weight":
            sd[key] = 1 + 0.1 * torch.randn(*shape, generator=g)
        elif key.endswith(".bias"):
            sd[key] = 0.1 * torch.randn(*shape, generator=g)
        else:
            sd[key] = torch.randn(*shape, generator=g) / shape[-1] ** 0.5
    C = block_channels(cfg)
    D = cfg.cross_attention_dim
    for i, b in processor_blocks(cfg).items():
        sd[f"ip_adapter.{i}.to_k_ip.weight"] = torch.randn(C[b], D, generator=g) / D ** 0.5
        sd[f"ip_adapter.{i}.to_v_ip.weight"] = torch.randn(C[b], D, generator=g) / D ** 0.5
    return sd


def default_encoder_config(base_cfg: UNetConfig):
    """The image encoder a base UNet's adapters were trained with: ViT-bigG/14 for SDXL, ViT-H/14 for SD v1.5; the tiny
    test UNets get the tiny test tower."""
    from . import vision_encoder as V
    if base_cfg.name.startswith("tiny"):
        return V.tiny_vision_config()
    return V.vit_bigg_config() if base_cfg.addition_embed_type == "text_time" else V.vit_h_config()


def plus_encoder_config(base_cfg: UNetConfig, embed_dim: Optional[int] = None):
    """The image encoder of a Plus adapter, chosen by the width E of the hidden states it reads (proj_in's
    in-features): ViT-H/14 (1280) for both SD v1.5 and SDXL, ViT-bigG/14 for 1664; None: ViT-H. The tiny test UNets
    get the tiny test tower."""
    from . import vision_encoder as V
    if base_cfg.name.startswith("tiny"):
        return V.tiny_vision_config()
    for c in (V.vit_h_config(), V.vit_bigg_config()):
        if embed_dim in (None, c.hidden_size):
            return c
    raise ValueError(f"image_proj.proj_in.weight: no default image encoder gives {embed_dim}-wide hidden states "
                     "(ViT-H/14: 1280, ViT-bigG/14: 1664); pass image_encoder=")


class IPAdapter:
    """One IP-Adapter for a base UNet, with its CLIP vision tower. `path_or_key` is a `.bin` / `.safetensors`
    checkpoint (a path with one of those suffixes that does not exist is an error), or any other key, which gets
    seeded synthetic weights: the plain projection, or with `image_proj="resampler"` an IP-Adapter Plus Resampler
    (`plus_geometry`). A checkpoint's kind follows from its keys (`is_resampler`); an `image_proj` given with a
    checkpoint must name that kind. `image_encoder` is an image-encoder
    directory (`config.json` + `model.safetensors`), or None for a seeded synthetic tower (`default_encoder_config` for
    the plain adapter, `plus_encoder_config` for Plus). The plain adapter's image embedding width must equal the tower's
    projection_dim, a Resampler's proj_in in-features the tower's hidden size."""

    def __init__(self, path_or_key: str, device, base_cfg: UNetConfig, image_encoder: Optional[str] = None,
                 n_tokens: int = 4, image_proj: Optional[str] = None):
        from . import vision_encoder as V
        if image_proj not in (None, "linear", "resampler"):
            raise ValueError(f"image_proj={image_proj!r}: 'linear' (IP-Adapter) or 'resampler' (IP-Adapter Plus)")
        if base_cfg.prediction_type != "epsilon" or base_cfg.name.split("_")[-1] not in ("sd15", "sdxl"):
            raise ValueError(f"IP-Adapter conditions SD v1.5 and SDXL UNets, not {base_cfg.name}")
        self.device = torch.device(device)
        seed = zlib.crc32(path_or_key.encode()) & 0x7FFFFFFF
        p = Path(path_or_key)
        sd = None
        if p.suffix in (".bin", ".safetensors"):
            if not p.is_file():
                raise FileNotFoundError(f"IP-Adapter checkpoint {path_or_key} does not exist")
            sd = read_ip_adapter_file(p)
        plus = is_resampler(sd) if sd is not None else image_proj == "resampler"
        if image_proj is not None and plus != (image_proj == "resampler"):
            raise ValueError(f"image_proj={image_proj!r}: {path_or_key} holds "
                             f"{'a Resampler (IP-Adapter Plus)' if plus else 'the plain linear projection'}")
        if image_encoder is not None:
            self.encoder_cfg, enc_sd = V.load_encoder_dir(image_encoder)
        else:
            E = sd["image_proj.proj_in.weight"].shape[1] if plus and sd is not None \
                and "image_proj.proj_in.weight" in sd else None
            self.encoder_cfg = plus_encoder_config(base_cfg, E) if plus else default_encoder_config(base_cfg)
            enc_sd = V.synthetic_state_dict(self.encoder_cfg, seed=zlib.crc32(f"{path_or_key}:encoder".encode())
                                            & 0x7FFFFFFF, device=self.device if self.device.type == "cuda" else "cpu")
        if sd is None:
            sd = (synthetic_ip_adapter_plus(base_cfg, plus_geometry(base_cfg, self.encoder_cfg.hidden_size), seed)
                  if plus else synthetic_ip_adapter(base_cfg, self.encoder_cfg.projection_dim, n_tokens, seed))
        self.key, self.base_cfg = path_or_key, base_cfg
        self.state_dict = sd
        if plus:
            self.weights, g = resampler_to_unet_keys(sd, base_cfg)
            if g["embed_dim"] != self.encoder_cfg.hidden_size:
                raise ValueError(f"image_proj.proj_in.weight: the Resampler takes {g['embed_dim']}-wide hidden states, "
                                 f"the image encoder gives {self.encoder_cfg.hidden_size}")
            self.resampler = {**g, "seq_len": self.encoder_cfg.num_positions}
            self.n_tokens, self.embed_dim = g["num_queries"], g["embed_dim"]
        else:
            self.resampler = None  # the plain Linear + LayerNorm projection
            self.weights, self.n_tokens, self.embed_dim = to_unet_keys(sd, base_cfg)
            if self.embed_dim != self.encoder_cfg.projection_dim:
                raise ValueError(f"image_proj.proj.weight: the adapter takes {self.embed_dim}-wide image embeddings, "
                                 f"the image encoder gives {self.encoder_cfg.projection_dim}")
        self._enc_sd = enc_sd
        self._encoder = None
        self._uncond = None

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
        prompt, or a sequence of `batch` of them -> the conditional rows on the device, fp16: image_embeds (batch, E),
        or for Plus the encoder's penultimate hidden states (batch, T, E)."""
        from . import vision_encoder as V
        if isinstance(images, torch.Tensor):
            t = images.detach().float().cpu()
            t = t.unsqueeze(0) if t.dim() == 3 else t
            images = [(x.clamp(0, 1).permute(1, 2, 0) * 255).round().to(torch.uint8).numpy() for x in t]
        elif not isinstance(images, (list, tuple)):
            images = [images]
        if len(images) not in (1, batch):
            raise ValueError(f"ip_adapter_image: {len(images)} images for {batch} prompts (give one, or one per prompt)")
        px = V.preprocess(images, self.encoder_cfg.image_size)
        e = self.encoder.encode_hidden(px, skip=1) if self.resampler else self.encoder.encode(px)
        return e.expand(batch, *e.shape[1:]).contiguous() if e.shape[0] == 1 else e

    def unconditional_hidden_states(self) -> torch.Tensor:
        """Plus: the encoder's penultimate hidden states of an all-zero preprocessed image (1, T, E) fp16, as diffusers'
        negative image embeds; computed once and cached."""
        if self._uncond is None:
            S = self.encoder_cfg.image_size
            self._uncond = self.encoder.encode_hidden(torch.zeros(1, 3, S, S), skip=1)
        return self._uncond

    def image_rows(self, hidden: torch.Tensor) -> torch.Tensor:
        """Plus: the 2 * batch rows the native handle takes for the conditional hidden states (batch, T, E), in
        cfgpp_set_prompt's order: the zero-pixel hidden states first, then `hidden`."""
        e = hidden.to(self.device, torch.float16)
        uc = self.unconditional_hidden_states().to(e.device)
        return torch.cat([uc.expand_as(e), e]).contiguous()

    def close(self):
        if self._encoder is not None:
            self._encoder.close()
            self._encoder = None
        self._uncond = None
