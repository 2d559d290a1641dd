"""ControlNet (diffusers `ControlNetModel`, guess_mode off) on the native backend: spatial conditioning of SD v1.5, SD 2.x
and SDXL trajectories by a control image (canny, depth, pose, scribble ... maps, made by the caller).

A ControlNet is a copy of the UNet's conv_in, time / add-embedding, down blocks and mid block with its own weights, plus
a small CNN on the control image (`controlnet_cond_embedding`) and one 1x1 "zero conv" per UNet skip tensor and one for
the mid block. The native handle runs it inside the UNet's fused step graph: its down / mid blocks are built by the
UNet executor's own block builders, and each zero conv adds its scaled output in place into the UNet's skip tensor (or
mid-block output) in the GEMM epilogue. See `cfgpp_attach_controlnet` in include/cfgpp_b200.h for the exact arithmetic.

`ControlNet(model_key | dir, device, base_cfg=...)` is the user-facing object: a diffusers ControlNetModel directory
(`config.json` + `diffusion_pytorch_model[.fp16].safetensors`) loads its weights; any other key gets seeded synthetic
weights for a ControlNet shaped like the base UNet (the offline stand-in, as for the UNets themselves).
"""
from __future__ import annotations

import ctypes
import json
import zlib
from ctypes import byref, c_int
from dataclasses import dataclass
from pathlib import Path
from typing import Dict, List, Optional, Tuple

import torch

from . import _native as nv
from .config import CFGPP_MAX_LEVELS, ModelDescExC, UNetConfig, to_desc
from .weights import Spec, synthetic_from_specs, unet_param_specs

CONDITIONING_EMBEDDING_CHANNELS = (16, 32, 96, 256)  # diffusers' default, used by every published SD / SDXL ControlNet
_CN_PREFIXES = ("conv_in.", "time_embedding.", "add_embedding.", "down_blocks.", "mid_block.")


@dataclass(frozen=True)
class ControlNetConfig:
    """`unet`: the ControlNet's own down / mid geometry in UNetConfig form (its up fields are unused);
    `conditioning_embedding_out_channels`: the control-image CNN's widths (it downsamples by 8)."""
    unet: UNetConfig
    conditioning_embedding_out_channels: Tuple[int, ...] = CONDITIONING_EMBEDDING_CHANNELS
    conditioning_channels: int = 3

    @property
    def residual_channels(self) -> List[int]:
        """Channels of the residual every zero conv produces, in `controlnet_down_blocks` order, then the mid block's."""
        boc, lpb = self.unet.block_out_channels, self.unet.layers_per_block
        out = [boc[0]]
        for i, c in enumerate(boc):
            out += [c] * lpb + ([c] if i != len(boc) - 1 else [])
        return out + [boc[-1]]


def controlnet_config(base: UNetConfig, **kw) -> ControlNetConfig:
    """A ControlNet shaped like the UNet `base` (as diffusers' `ControlNetModel.from_unet` makes one)."""
    return ControlNetConfig(unet=base, **kw)


def config_from_diffusers(cfg: dict, name: str = "controlnet") -> ControlNetConfig:
    """The ControlNetConfig of a diffusers ControlNetModel `config.json` (as a dict). Refuses what the native ControlNet
    does not run: global_pool_conditions, a channel order other than rgb, conditioning_channels other than 3."""
    if cfg.get("global_pool_conditions", False):
        raise ValueError("global_pool_conditions ControlNets are not supported")
    if cfg.get("controlnet_conditioning_channel_order", "rgb") != "rgb":
        raise ValueError(f"controlnet_conditioning_channel_order {cfg['controlnet_conditioning_channel_order']!r}: "
                         "only 'rgb' is supported")
    if cfg.get("conditioning_channels", 3) != 3:
        raise ValueError(f"conditioning_channels {cfg['conditioning_channels']}: only 3 (RGB control images)")
    boc = tuple(cfg.get("block_out_channels", (320, 640, 1280, 1280)))
    L = len(boc)

    def per_level(v, default):
        v = default if v is None else v
        return tuple(v) if isinstance(v, (list, tuple)) else (v,) * L

    down = tuple(cfg.get("down_block_types", ("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",)))
    up = tuple("CrossAttnUpBlock2D" if t == "CrossAttnDownBlock2D" else "UpBlock2D" for t in reversed(down))
    # diffusers: num_attention_heads falls back to attention_head_dim (which names the head count there)
    heads = per_level(cfg.get("num_attention_heads") or cfg.get("attention_head_dim"), 8)
    add_type = cfg.get("addition_embed_type")
    ate = cfg.get("addition_time_embed_dim") or 256
    proj = cfg.get("projection_class_embeddings_input_dim") or 2816
    unet = UNetConfig(
        name=name, sample_size=cfg.get("sample_size") or 64, in_channels=cfg.get("in_channels", 4),
        block_out_channels=boc, down_block_types=down, up_block_types=up,
        layers_per_block=cfg.get("layers_per_block", 2),
        transformer_layers_per_block=per_level(cfg.get("transformer_layers_per_block"), 1),
        num_attention_heads=heads, cross_attention_dim=cfg.get("cross_attention_dim", 768),
        use_linear_projection=bool(cfg.get("use_linear_projection", False)),
        norm_num_groups=cfg.get("norm_num_groups", 32), norm_eps=cfg.get("norm_eps", 1e-5),
        addition_embed_type=add_type, addition_time_embed_dim=ate, projection_class_embeddings_input_dim=proj,
        # SDXL text_time: pooled text embeds + 6 time ids
        pooled_dim=proj - 6 * ate if add_type == "text_time" else 1280)
    return ControlNetConfig(unet=unet, conditioning_embedding_out_channels=tuple(
        cfg.get("conditioning_embedding_out_channels", CONDITIONING_EMBEDDING_CHANNELS)), conditioning_channels=3)


def controlnet_param_specs(cfg: ControlNetConfig) -> List[Spec]:
    """Every parameter of ControlNetModel(cfg) in diffusers naming, with its shape and synthetic-weight kind."""
    out = [s for s in unet_param_specs(cfg.unet) if s[0].startswith(_CN_PREFIXES)]
    ch = cfg.conditioning_embedding_out_channels
    e = "controlnet_cond_embedding"
    out += [(f"{e}.conv_in.weight", (ch[0], cfg.conditioning_channels, 3, 3), "w"), (f"{e}.conv_in.bias", (ch[0],), "b")]
    for i in range(len(ch) - 1):
        out += [(f"{e}.blocks.{2 * i}.weight", (ch[i], ch[i], 3, 3), "w"), (f"{e}.blocks.{2 * i}.bias", (ch[i],), "b"),
                (f"{e}.blocks.{2 * i + 1}.weight", (ch[i + 1], ch[i], 3, 3), "w"),
                (f"{e}.blocks.{2 * i + 1}.bias", (ch[i + 1],), "b")]
    c0 = cfg.unet.block_out_channels[0]
    out += [(f"{e}.conv_out.weight", (c0, ch[-1], 3, 3), "w"), (f"{e}.conv_out.bias", (c0,), "b")]
    res = cfg.residual_channels
    for k, c in enumerate(res[:-1]):
        out += [(f"controlnet_down_blocks.{k}.weight", (c, c, 1, 1), "w"), (f"controlnet_down_blocks.{k}.bias", (c,), "b")]
    out += [("controlnet_mid_block.weight", (res[-1], res[-1], 1, 1), "w"), ("controlnet_mid_block.bias", (res[-1],), "b")]
    return out


def synthetic_controlnet_state_dict(cfg: ControlNetConfig, seed: int = 4321, device="cpu",
                                    dtype=torch.float16) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights in weights.py's style. The zero convs are random and non-zero, as in a trained
    ControlNet (zeros would make every comparison with and without the ControlNet vacuous)."""
    return synthetic_from_specs(controlnet_param_specs(cfg), seed, device, dtype)


def control_scales(num_steps: int, scale: float = 1.0, start: float = 0.0, end: float = 1.0,
                   entries_per_step: int = 1, first: int = 0, count: Optional[int] = None) -> List[float]:
    """The conditioning scale of every schedule entry, by diffusers' control_guidance_start / end rule:
    s_i = scale * (1 - [i / N < start or (i + 1) / N > end]) for sampler step i of N. A DPM-Solver++(2S) step has two
    schedule entries (entries_per_step = 2) that share their step's s_i. `first` / `count` select the steps one handle
    runs when a trajectory is split between two UNets (the indices run over the whole schedule)."""
    count = num_steps - first if count is None else count
    out = []
    for i in range(first, first + count):
        keep = 1.0 - float(i / num_steps < start or (i + 1) / num_steps > end)
        out += [scale * keep] * entries_per_step
    return out


def entry_steps(steps) -> List[int]:
    """The sampler step each schedule entry belongs to: the two entries of a DPM-Solver++(2S) step (midpoint, then the
    final entry, second_order bit 32) share one step, every other entry is a step of its own."""
    from .schedule import KD_2S_FINAL
    out, i = [], -1
    for st in steps:
        if not (st.coef.second_order & KD_2S_FINAL):
            i += 1
        out.append(max(i, 0))
    return out


def entry_scales(steps, scale: float = 1.0, start: float = 0.0, end: float = 1.0) -> List[float]:
    """control_scales over a schedule's entries: N = the schedule's sampler steps, whichever engine runs which entries
    (a refiner hand-off splits the entries, not the indices)."""
    idx = entry_steps(steps)
    per_step = control_scales(idx[-1] + 1 if idx else 0, scale, start, end)
    return [per_step[i] for i in idx]


@dataclass
class ControlRequest:
    """What one sample() call asks of the ControlNet: the handle, the control image on the engine's device
    (batch, 3, H, W), and the diffusers scale rule's parameters."""
    engine: "NativeControlNet"
    image: torch.Tensor
    scale: float = 1.0
    start: float = 0.0
    end: float = 1.0

    def step_scale(self, i: int, n: int) -> float:
        return control_scales(n, self.scale, self.start, self.end, first=i, count=1)[0]

    def entry_scales(self, steps) -> List[float]:
        return entry_scales(steps, self.scale, self.start, self.end)


def control_request(kwargs: dict, batch: int, height: int, width: int, device) -> Optional[ControlRequest]:
    """The ControlRequest of a text-to-image sample() call's keyword arguments (controlnet=, control_image=,
    controlnet_conditioning_scale=, control_guidance_start=, control_guidance_end=), or None without controlnet=.
    Raises ValueError on a missing or mis-sized control image or an empty guidance window."""
    cn = kwargs.get("controlnet")
    image = kwargs.get("control_image")
    if cn is None:
        if image is not None:
            raise ValueError("control_image given without controlnet=")
        return None
    if image is None:
        raise ValueError("controlnet= needs control_image=")
    start = float(kwargs.get("control_guidance_start", 0.0))
    end = float(kwargs.get("control_guidance_end", 1.0))
    if not 0.0 <= start < end <= 1.0:
        raise ValueError(f"control_guidance_start / end must satisfy 0 <= start < end <= 1 (got {start}, {end})")
    engine = cn.engine if isinstance(cn, ControlNet) else cn
    if not isinstance(engine, NativeControlNet):
        raise ValueError("controlnet= takes a cfgpp_b200.controlnet.ControlNet")
    image = check_control_image(image, batch, height, width).to(device).contiguous()
    return ControlRequest(engine, image, float(kwargs.get("controlnet_conditioning_scale", 1.0)), start, end)


class ControlNetDescC(ctypes.Structure):
    """`cfgpp_controlnet_desc` of include/cfgpp_b200.h."""
    _fields_ = [("model", ModelDescExC), ("conditioning_channels", c_int), ("num_embedding_levels", c_int),
                ("embedding_channels", c_int * CFGPP_MAX_LEVELS)]


def to_controlnet_desc(cfg: ControlNetConfig) -> ControlNetDescC:
    ch = cfg.conditioning_embedding_out_channels
    if len(ch) != 4:
        raise ValueError("the conditioning embedding must take 4 channel counts (it downsamples by 8)")
    d = ControlNetDescC()
    d.model = to_desc(cfg.unet)
    d.model.prediction_type = 0
    d.conditioning_channels = cfg.conditioning_channels
    d.num_embedding_levels = len(ch)
    for i, c in enumerate(ch):
        d.embedding_channels[i] = c
    return d


class NativeControlNet(nv.NativeHandle):
    """Owner of one native ControlNet handle (cfgpp_controlnet_create). It runs through the NativeUNet it is attached
    to (NativeUNet.attach_controlnet)."""
    _prefix, _what = "", "ControlNet"

    def __init__(self, cfg: ControlNetConfig, state_dict: Dict[str, torch.Tensor], device="cuda:0"):
        self.cfg = cfg
        self.attached_to = None
        self._open(to_controlnet_desc(cfg), state_dict.items(), device)

    def _create(self, desc, idx: int) -> None:
        nv.check(self.lib.cfgpp_controlnet_create(byref(desc), c_int(idx), byref(self._h)))

    def close(self):
        if getattr(self, "attached_to", None) is not None:  # the UNet engine's plan reads this handle: detach first
            self.attached_to.attach_controlnet(None)
        super().close()

    def embed(self, image: torch.Tensor) -> torch.Tensor:
        """The conditioning embedding alone: image (B, 3, H, W) in [0, 1] -> (B, H/8, W/8, C0) NHWC fp16."""
        image = image.to(self.device).contiguous()
        B, _, H, W = image.shape
        out = torch.empty((B, H // 8, W // 8, self.cfg.unet.block_out_channels[0]), dtype=torch.float16,
                          device=self.device)
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_controlnet_embed(self._h, nv.ptr(image), c_int(nv.dtype_code(image)), c_int(B),
                                                     c_int(H), c_int(W), nv.ptr(out), nv.stream_ptr()))
        return out


def load_controlnet_dir(path, device="cpu", dtype=torch.float16):
    """(ControlNetConfig, state dict) of a diffusers ControlNetModel directory."""
    from .checkpoints import find_controlnet_files
    from .weights import load_safetensors_state_dict
    files = find_controlnet_files(path)
    cfg = config_from_diffusers(json.loads(files["config"].read_text()), name=Path(path).name or "controlnet")
    return cfg, load_safetensors_state_dict(str(files["weights"]), device, dtype)


class ControlNet:
    """A ControlNet for the solvers of one model family. `model_key`: a diffusers ControlNetModel directory, or a name
    that gets seeded synthetic weights shaped like `base_cfg` (the base UNet's config). `state_dict` / `config` override
    what the key would load."""

    def __init__(self, model_key: str = "controlnet", device="cuda", base_cfg: Optional[UNetConfig] = None,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, config: Optional[ControlNetConfig] = None):
        if config is None and state_dict is None and Path(model_key).is_dir():
            config, state_dict = load_controlnet_dir(model_key)
        if config is None:
            if base_cfg is None:
                raise ValueError("a synthetic ControlNet needs base_cfg (the UNet config it conditions)")
            config = controlnet_config(base_cfg)
        if state_dict is None:
            state_dict = synthetic_controlnet_state_dict(config, seed=zlib.crc32(model_key.encode()) & 0x7FFFFFFF)
        self.cfg = config
        self.engine = NativeControlNet(config, state_dict, device)

    def embed(self, image: torch.Tensor) -> torch.Tensor:
        return self.engine.embed(image)


def check_control_image(image: torch.Tensor, batch: int, height: int, width: int) -> torch.Tensor:
    """`image` (B, 3, H, W) or (1, 3, H, W), broadcast over the batch, at exactly the output size (no resizing).
    Returns the (batch, 3, height, width) tensor. Raises ValueError otherwise."""
    if not torch.is_tensor(image) or image.dim() != 4 or image.shape[1] != 3:
        raise ValueError("control_image must be a (B, 3, H, W) tensor")
    if tuple(image.shape[2:]) != (height, width):
        raise ValueError(f"control_image is {tuple(image.shape[2:])}, the output is {(height, width)}: "
                         "it is not resized, pass it at the output size")
    if image.shape[0] not in (1, batch):
        raise ValueError(f"control_image has {image.shape[0]} images for a batch of {batch}")
    return image.expand(batch, -1, -1, -1)


__all__ = ["ControlNet", "ControlNetConfig", "ControlRequest", "NativeControlNet", "check_control_image",
           "config_from_diffusers", "control_request", "control_scales", "entry_scales", "entry_steps", "controlnet_config", "controlnet_param_specs", "synthetic_controlnet_state_dict"]
