"""CLIP vision tower (transformers `CLIPVisionModelWithProjection`) on the native library, and CLIPImageProcessor's
preprocessing on the host: the image encoder of IP-Adapter (ViT-H/14 for SD v1.5's adapter, ViT-bigG/14 for SDXL's).
No transformers import: the configuration is read from the encoder directory's `config.json` and the weights from its
`model.safetensors`."""
from __future__ import annotations

import ctypes
import json
import math
from ctypes import byref, c_double, c_int, c_size_t
from dataclasses import dataclass
from pathlib import Path
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _native as nv

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


@dataclass(frozen=True)
class CLIPVisionConfig:
    hidden_size: int = 1280
    intermediate_size: int = 5120
    num_hidden_layers: int = 32
    num_attention_heads: int = 16
    image_size: int = 224
    patch_size: int = 14
    hidden_act: str = "gelu"
    projection_dim: int = 1024
    layer_norm_eps: float = 1e-5

    @property
    def num_positions(self) -> int:
        return (self.image_size // self.patch_size) ** 2 + 1


def vit_h_config() -> CLIPVisionConfig:
    """IP-Adapter's `models/image_encoder` (OpenCLIP ViT-H/14): heads of 80."""
    return CLIPVisionConfig()


def vit_bigg_config() -> CLIPVisionConfig:
    """IP-Adapter's `sdxl_models/image_encoder` (OpenCLIP ViT-bigG/14): heads of 104."""
    return CLIPVisionConfig(hidden_size=1664, intermediate_size=8192, num_hidden_layers=48, projection_dim=1280)


def tiny_vision_config(projection_dim: int = 64) -> CLIPVisionConfig:
    """Test geometry: 2 layers, heads of 80 (padded to 128), 8x8 patches of a 32-pixel image (17 tokens)."""
    return CLIPVisionConfig(hidden_size=320, intermediate_size=640, num_hidden_layers=2, num_attention_heads=4,
                            image_size=32, patch_size=8, projection_dim=projection_dim)


def config_from_json(cfg: dict) -> CLIPVisionConfig:
    v = cfg.get("vision_config", cfg)
    fields = {f: v[f] for f in CLIPVisionConfig.__dataclass_fields__ if f in v}
    if "projection_dim" in cfg and "projection_dim" not in v:
        fields["projection_dim"] = cfg["projection_dim"]
    return CLIPVisionConfig(**fields)


class ClipVisionDescC(ctypes.Structure):
    _fields_ = [("hidden_size", c_int), ("intermediate_size", c_int), ("num_layers", c_int), ("num_heads", c_int),
                ("image_size", c_int), ("patch_size", c_int), ("hidden_act", c_int), ("projection_dim", c_int),
                ("layer_norm_eps", ctypes.c_float)]


def to_desc(cfg: CLIPVisionConfig) -> ClipVisionDescC:
    acts = {"quick_gelu": 0, "gelu": 1}
    if cfg.hidden_act not in acts:
        raise ValueError(f"hidden_act {cfg.hidden_act!r}: quick_gelu or gelu")
    return ClipVisionDescC(cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers, cfg.num_attention_heads,
                           cfg.image_size, cfg.patch_size, acts[cfg.hidden_act], cfg.projection_dim, cfg.layer_norm_eps)


def param_specs(cfg: CLIPVisionConfig) -> List[Tuple[str, Tuple[int, ...], str]]:
    D, I, P = cfg.hidden_size, cfg.intermediate_size, cfg.patch_size
    vm = "vision_model."
    specs = [(vm + "embeddings.class_embedding", (D,), "emb"),
             (vm + "embeddings.patch_embedding.weight", (D, 3, P, P), "w"),
             (vm + "embeddings.position_embedding.weight", (cfg.num_positions, D), "pos"),
             (vm + "pre_layrnorm.weight", (D,), "norm_w"), (vm + "pre_layrnorm.bias", (D,), "norm_b")]
    for l in range(cfg.num_hidden_layers):
        p = f"{vm}encoder.layers.{l}."
        for n in ("q_proj", "k_proj", "v_proj"):
            specs += [(p + f"self_attn.{n}.weight", (D, D), "w"), (p + f"self_attn.{n}.bias", (D,), "b")]
        specs += [(p + "self_attn.out_proj.weight", (D, D), "w_res"), (p + "self_attn.out_proj.bias", (D,), "b"),
                  (p + "layer_norm1.weight", (D,), "norm_w"), (p + "layer_norm1.bias", (D,), "norm_b"),
                  (p + "mlp.fc1.weight", (I, D), "w"), (p + "mlp.fc1.bias", (I,), "b"),
                  (p + "mlp.fc2.weight", (D, I), "w_res"), (p + "mlp.fc2.bias", (D,), "b"),
                  (p + "layer_norm2.weight", (D,), "norm_w"), (p + "layer_norm2.bias", (D,), "norm_b")]
    specs += [(vm + "post_layernorm.weight", (D,), "norm_w"), (vm + "post_layernorm.bias", (D,), "norm_b"),
              ("visual_projection.weight", (cfg.projection_dim, D), "w")]
    return specs


def synthetic_state_dict(cfg: CLIPVisionConfig, seed: int = 555, device="cpu",
                         dtype=torch.float16) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights (activation-preserving scales, residual branches damped by depth)."""
    g = torch.Generator(device=device).manual_seed(seed)
    damp = 1.0 / math.sqrt(2.0 * cfg.num_hidden_layers)
    sd = {}
    for key, shape, kind in param_specs(cfg):
        if kind == "norm_w":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        elif kind in ("norm_b", "b"):
            t = 0.02 * torch.randn(shape, generator=g, device=device)
        elif kind == "emb":
            t = 0.5 * torch.randn(shape, generator=g, device=device)
        elif kind == "pos":
            t = 0.25 * torch.randn(shape, generator=g, device=device)
        else:
            gain = 1.0 if kind == "w" else 2.0 * damp
            t = torch.randn(shape, generator=g, device=device) * (gain / math.sqrt(math.prod(shape[1:])))
        sd[key] = t.to(dtype)
    return sd


def load_encoder_dir(path) -> Tuple[CLIPVisionConfig, Dict[str, torch.Tensor]]:
    """An image-encoder directory: `config.json` + `model.safetensors` (transformers' layout)."""
    from safetensors.torch import load_file
    path = Path(path)
    for f in ("config.json", "model.safetensors"):
        if not (path / f).is_file():
            raise ValueError(f"{path}: image-encoder directory lacks {f}")
    cfg = config_from_json(json.loads((path / "config.json").read_text()))
    sd = {k: v for k, v in load_file(str(path / "model.safetensors")).items() if k != "vision_model.embeddings.position_ids"}
    return cfg, sd


def preprocess(images: Sequence, size: int = 224) -> torch.Tensor:
    """CLIPImageProcessor's steps on the host: resize the shortest side to `size` (PIL bicubic), center crop
    size x size, x 1/255, normalise by CLIP's mean and std. `images`: PIL images, or uint8 arrays (H, W, 3).
    Returns pixel values (n, 3, size, size) fp32."""
    from PIL import Image
    out = []
    for im in images:
        if not isinstance(im, Image.Image):
            im = Image.fromarray(np.asarray(im, dtype=np.uint8))
        im = im.convert("RGB")
        w, h = im.size
        short, long = (w, h) if w <= h else (h, w)
        new_long = int(size * long / short)
        nw, nh = (size, new_long) if w <= h else (new_long, size)
        im = im.resize((nw, nh), Image.BICUBIC)
        top, left = (nh - size) // 2, (nw - size) // 2
        a = (np.asarray(im, dtype=np.uint8)[top:top + size, left:left + size].astype(np.float64) / 255).astype(np.float32)
        a = (a - np.array(CLIP_MEAN, dtype=np.float32)) / np.array(CLIP_STD, dtype=np.float32)
        out.append(torch.from_numpy(np.ascontiguousarray(a.transpose(2, 0, 1))))
    return torch.stack(out)


class NativeCLIPVisionEncoder(nv.NativeHandle):
    """Owner of one `cfgpp_clip_vision_handle`: `encode(pixel_values)` -> image_embeds (n, projection_dim) fp16, and
    `encode_hidden(pixel_values, skip)` -> hidden_states[num_layers - skip] (n, T, hidden_size) fp16."""

    _prefix, _what = "_clip_vision", "vision encoder"

    def __init__(self, cfg: CLIPVisionConfig, state_dict: Dict[str, torch.Tensor], device="cuda:0"):
        self.cfg = cfg

        def weights():
            for key, shape, _ in param_specs(cfg):
                if key not in state_dict:
                    raise ValueError(f"CLIP vision state dict lacks '{key}'")
                w = state_dict[key]
                if tuple(w.shape) != tuple(shape):
                    raise ValueError(f"{key}: shape {tuple(w.shape)} != {tuple(shape)}")
                yield key, (w if w.dtype in (torch.float16, torch.float32) else w.float())

        self._open(to_desc(cfg), weights(), device)

    def encode(self, pixel_values: torch.Tensor) -> torch.Tensor:
        n, S = pixel_values.shape[0], self.cfg.image_size
        assert tuple(pixel_values.shape[1:]) == (3, S, S), "pixel values (n, 3, image_size, image_size)"
        x = pixel_values.to(self.device).contiguous()
        outs = []
        with torch.cuda.device(self.device):
            for i in range(0, n, 16):
                xi = x[i:i + 16]
                out = torch.empty((xi.shape[0], self.cfg.projection_dim), dtype=torch.float16, device=self.device)
                nv.check(self.lib.cfgpp_clip_vision_encode(self._h, nv.ptr(xi), c_int(nv.dtype_code(xi)),
                                                           c_int(xi.shape[0]), nv.ptr(out), nv.stream_ptr()))
                outs.append(out)
        return torch.cat(outs)

    def encode_hidden(self, pixel_values: torch.Tensor, skip: int = 1) -> torch.Tensor:
        """hidden_states[num_layers - skip] of transformers' `output_hidden_states=True` (skip = 1: hidden_states[-2],
        what IP-Adapter Plus reads; skip = 0: the last layer's output, before post_layernorm)."""
        n, S = pixel_values.shape[0], self.cfg.image_size
        assert tuple(pixel_values.shape[1:]) == (3, S, S), "pixel values (n, 3, image_size, image_size)"
        x = pixel_values.to(self.device).contiguous()
        T = self.cfg.num_positions
        out = torch.empty((n, T, self.cfg.hidden_size), dtype=torch.float16, device=self.device)
        with torch.cuda.device(self.device):
            for i in range(0, n, 16):
                xi = x[i:i + 16]
                nv.check(self.lib.cfgpp_clip_vision_encode_hidden(self._h, nv.ptr(xi), c_int(nv.dtype_code(xi)),
                                                                  c_int(xi.shape[0]), c_int(skip), nv.ptr(out[i:i + 16]),
                                                                  nv.stream_ptr()))
        return out

    @property
    def stats(self) -> dict:
        f, w = c_double(), c_size_t()
        nv.check(self.lib.cfgpp_clip_vision_stats(self._h, byref(f), byref(w)))
        return {"flops": f.value, "workspace_bytes": w.value}
