"""T2I-Adapter (Mou et al. 2023; diffusers `T2IAdapter`, `full_adapter` / `full_adapter_xl`) on the native backend:
spatial conditioning of SD v1.5, SD 2.x and SDXL trajectories by a conditioning image (canny, sketch, lineart, depth,
openpose maps made by the caller), at almost no per-step cost.

The adapter is a small CNN that runs once per image (`NativeT2IAdapter`, csrc/t2i_adapter.cu) and gives four feature
maps. The UNet handle adds them into its down path inside the fused step graph, one gated launch per feature, at the
placements of diffusers' `down_intrablock_additional_residuals` (see `cfgpp_t2i_attach` in include/cfgpp_b200.h). A
per-entry word of the step record switches the adds off after `adapter_conditioning_factor` of the sampler steps.

`T2IAdapter(model_key | dir, device, base_cfg=...)` is the user-facing object: a diffusers T2IAdapter directory
(`config.json` + `diffusion_pytorch_model[.fp16].safetensors`) loads its weights; any other key gets seeded synthetic
weights for an adapter shaped like the base UNet (the offline stand-in, as for the UNets themselves). Pass it to any
text-to-image solver's `sample(t2i_adapter=..., t2i_adapter_image=...)`. ("t2i" names it throughout: "adapter" alone
means a LoRA adapter in lora.py and the C ABI.)
"""
from __future__ import annotations

import ctypes
import json
import zlib
from ctypes import byref, c_float, c_int, c_void_p
from dataclasses import dataclass
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _native as nv
from .config import UNetConfig
from .weights import Spec, synthetic_from_specs

KINDS = {"full_adapter": 0, "full_adapter_xl": 1}


@dataclass(frozen=True)
class T2IAdapterConfig:
    """diffusers `T2IAdapter(adapter_type, in_channels, channels, num_res_blocks, downscale_factor)`."""
    adapter_type: str = "full_adapter"
    in_channels: int = 3
    channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    num_res_blocks: int = 2
    downscale_factor: int = 8

    def blocks(self) -> List[Tuple[int, int, bool]]:
        """(in, out, down) of every AdapterBlock: FullAdapter (c0,c0), (c[i-1],c[i],down); FullAdapterXL (c0,c0),
        (c0,c1), (c1,c2,down), (c3,c3)."""
        c = self.channels
        if self.adapter_type == "full_adapter":
            return [(c[0], c[0], False)] + [(c[i - 1], c[i], True) for i in range(1, len(c))]
        return [(c[0], c[0], False), (c[0], c[1], False), (c[1], c[2], True), (c[3], c[3], False)]

    @property
    def total_downscale_factor(self) -> int:
        """The side every adapter image must be a multiple of (diffusers rounds its default size to it)."""
        return self.downscale_factor * (2 ** (len(self.channels) - 1) if self.adapter_type == "full_adapter" else 2)

    def feature_shapes(self, height: int, width: int) -> List[Tuple[int, int, int]]:
        """(C, h, w) of every feature of an adapter image (height, width)."""
        h, w = height // self.downscale_factor, width // self.downscale_factor
        out = []
        for _, cout, down in self.blocks():
            if down:
                h, w = h // 2, w // 2
            out.append((cout, h, w))
        return out


def config_from_diffusers(cfg: dict) -> T2IAdapterConfig:
    """The T2IAdapterConfig of a diffusers T2IAdapter `config.json` (as a dict). Refuses what the native adapter does not
    run: `light_adapter`, a MultiAdapter and any other adapter type."""
    cls = cfg.get("_class_name", "T2IAdapter")
    if cls != "T2IAdapter":
        raise ValueError(f"{cls}: only a single T2IAdapter is supported (MultiAdapter is not)")
    kind = cfg.get("adapter_type", "full_adapter")
    if kind not in KINDS:
        raise ValueError(f"adapter_type {kind!r}: only 'full_adapter' and 'full_adapter_xl' are supported")
    out = T2IAdapterConfig(adapter_type=kind, in_channels=int(cfg.get("in_channels", 3)),
                           channels=tuple(cfg.get("channels", (320, 640, 1280, 1280))),
                           num_res_blocks=int(cfg.get("num_res_blocks", 2)),
                           downscale_factor=int(cfg.get("downscale_factor", 8 if kind == "full_adapter" else 16)))
    if out.in_channels not in (1, 3):
        raise ValueError(f"in_channels {out.in_channels}: a T2I-Adapter image has 1 or 3 channels")
    if len(out.channels) != 4:
        raise ValueError(f"channels {out.channels}: the native adapter takes 4 blocks")
    if kind == "full_adapter_xl" and out.channels[2] != out.channels[3]:
        raise ValueError(f"full_adapter_xl channels {out.channels}: channels[3] must equal channels[2]")
    return out


def t2i_adapter_config(base: UNetConfig, in_channels: int = 3) -> T2IAdapterConfig:
    """An adapter shaped for the UNet `base`: full_adapter_xl (factor 16) for an SDXL-style UNet (text_time
    add-embedding), full_adapter (factor 8) otherwise."""
    boc = tuple(base.block_out_channels)
    if base.addition_embed_type == "text_time":
        return T2IAdapterConfig("full_adapter_xl", in_channels, boc + (boc[-1],), 2, 16)
    return T2IAdapterConfig("full_adapter", in_channels, boc, 2, 8)


def t2i_adapter_param_specs(cfg: T2IAdapterConfig) -> List[Spec]:
    """Every parameter of T2IAdapter(cfg) in diffusers naming (`adapter.*`), with its shape and synthetic-weight kind."""
    cu = cfg.in_channels * cfg.downscale_factor ** 2
    out: List[Spec] = [("adapter.conv_in.weight", (cfg.channels[0], cu, 3, 3), "w"),
                       ("adapter.conv_in.bias", (cfg.channels[0],), "b")]
    for i, (cin, cout, _) in enumerate(cfg.blocks()):
        p = f"adapter.body.{i}"
        if cin != cout:
            out += [(f"{p}.in_conv.weight", (cout, cin, 1, 1), "w"), (f"{p}.in_conv.bias", (cout,), "b")]
        for j in range(cfg.num_res_blocks):
            r = f"{p}.resnets.{j}"
            out += [(f"{r}.block1.weight", (cout, cout, 3, 3), "w"), (f"{r}.block1.bias", (cout,), "b"),
                    (f"{r}.block2.weight", (cout, cout, 1, 1), "w_res"), (f"{r}.block2.bias", (cout,), "b")]
    return out


def synthetic_t2i_adapter_state_dict(cfg: T2IAdapterConfig, seed: int = 4321, device="cpu",
                                     dtype=torch.float16) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights in weights.py's style."""
    return synthetic_from_specs(t2i_adapter_param_specs(cfg), seed, device, dtype)


def unet_placements(ucfg: UNetConfig, h_lat: int, w_lat: int) -> List[Tuple[int, int, int]]:
    """(C, h, w) of the tensor each feature lands on, in order: per down block the last (resnet, attention) output of a
    CrossAttnDownBlock2D or the (downsampled) output of a DownBlock2D, then the mid-block output."""
    boc, L = ucfg.block_out_channels, len(ucfg.block_out_channels)
    out = []
    for i in range(L):
        s = 2 ** i if ucfg.down_block_types[i] == "CrossAttnDownBlock2D" or i == L - 1 else 2 ** (i + 1)
        out.append((boc[i], h_lat // s, w_lat // s))
    return out + [(boc[-1], h_lat // 2 ** (L - 1), w_lat // 2 ** (L - 1))]


def check_placements(cfg: T2IAdapterConfig, ucfg: UNetConfig, height: int, width: int) -> None:
    """Raises ValueError unless the adapter's features of a (height, width) image are, in order, the shapes of the
    UNet tensors they land on (all down placements, then the mid-block output for a feature left over)."""
    feats = cfg.feature_shapes(height, width)
    places = unet_placements(ucfg, height // ucfg.vae_scale_factor, width // ucfg.vae_scale_factor)
    L = len(ucfg.block_out_channels)
    if len(feats) not in (L, L + 1) or feats != places[:len(feats)]:
        raise ValueError(f"the T2I-Adapter ({cfg.adapter_type}, channels {cfg.channels}) gives features {feats} at "
                         f"{width}x{height}; {ucfg.name} takes {places[:L]} (+ mid {places[L]})")


def step_flags(num_steps: int, factor: float) -> List[bool]:
    """diffusers' adapter_conditioning_factor rule: the features are added at sampler step i of N while
    i < int(N * factor)."""
    cut = int(num_steps * factor)
    return [i < cut for i in range(num_steps)]


def entry_flags(steps, factor: float) -> List[bool]:
    """step_flags over a schedule's entries (the two entries of a DPM-Solver++(2S) step share one flag); N is the whole
    schedule's step count, so an engine that runs part of the entries (a refiner hand-off) keeps its indices."""
    from .controlnet import entry_steps
    idx = entry_steps(steps)
    per_step = step_flags(idx[-1] + 1 if idx else 0, factor)
    return [per_step[i] for i in idx]


class T2IAdapterDescC(ctypes.Structure):
    """`cfgpp_t2i_adapter_desc` of include/cfgpp_b200.h."""
    _fields_ = [("kind", c_int), ("in_channels", c_int), ("channels", c_int * 4), ("num_res_blocks", c_int),
                ("downscale_factor", c_int)]


def to_t2i_adapter_desc(cfg: T2IAdapterConfig) -> T2IAdapterDescC:
    d = T2IAdapterDescC()
    d.kind = KINDS[cfg.adapter_type]
    d.in_channels = cfg.in_channels
    for i, c in enumerate(cfg.channels):
        d.channels[i] = c
    d.num_res_blocks = cfg.num_res_blocks
    d.downscale_factor = cfg.downscale_factor
    return d


class NativeT2IAdapter(nv.NativeHandle):
    """Owner of one native T2I-Adapter handle (cfgpp_t2i_adapter_create)."""
    _prefix, _what = "_t2i_adapter", "T2I-Adapter"

    def __init__(self, cfg: T2IAdapterConfig, state_dict: Dict[str, torch.Tensor], device="cuda:0"):
        self.cfg = cfg
        self._open(to_t2i_adapter_desc(cfg), state_dict.items(), device)

    def features(self, image: torch.Tensor, scale: float = 1.0) -> List[torch.Tensor]:
        """image (B, in_channels, H, W) in [0, 1] (fp16 or fp32) -> the features, each (B, h, w, C) NHWC fp16, already
        multiplied by `scale` in fp16."""
        image = image.to(self.device).contiguous()
        B, _, H, W = image.shape
        outs = [torch.empty((B, h, w, c), dtype=torch.float16, device=self.device)
                for c, h, w in self.cfg.feature_shapes(H, W)]
        ptrs = (c_void_p * len(outs))(*[o.data_ptr() for o in outs])
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_t2i_adapter_forward(self._h, nv.ptr(image), c_int(nv.dtype_code(image)), c_int(B),
                                                        c_int(H), c_int(W), c_float(float(scale)), ptrs,
                                                        nv.stream_ptr()))
        return outs

    @property
    def stats(self) -> dict:
        """{'flops', 'workspace_bytes'} of the last prepared forward."""
        f, b = ctypes.c_double(), ctypes.c_size_t()
        nv.check(self.lib.cfgpp_t2i_adapter_stats(self._h, byref(f), byref(b)))
        return {"flops": f.value, "workspace_bytes": b.value}


def load_t2i_adapter_dir(path, device="cpu", dtype=torch.float16):
    """(T2IAdapterConfig, state dict) of a diffusers T2IAdapter directory."""
    from .checkpoints import find_t2i_adapter_files
    from .weights import load_safetensors_state_dict
    files = find_t2i_adapter_files(path)
    cfg = config_from_diffusers(json.loads(files["config"].read_text()))
    return cfg, load_safetensors_state_dict(str(files["weights"]), device, dtype)


class T2IAdapter:
    """A T2I-Adapter for the solvers of one UNet. `model_key`: a diffusers T2IAdapter directory, or a name that gets
    seeded synthetic weights shaped for `base_cfg` (with `in_channels` 3, or 1 for a sketch / canny adapter).
    `state_dict` / `config` override what the key would load. Raises ValueError when the features do not land on
    `base_cfg`'s down path."""

    def __init__(self, model_key: str = "t2i_adapter", device="cuda", base_cfg: Optional[UNetConfig] = None,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, config: Optional[T2IAdapterConfig] = None,
                 in_channels: int = 3):
        if base_cfg is None:
            raise ValueError("a T2I-Adapter needs base_cfg (the UNet config it conditions)")
        if config is None and state_dict is None and Path(model_key).is_dir():
            config, state_dict = load_t2i_adapter_dir(model_key)
        if config is None:
            config = t2i_adapter_config(base_cfg, in_channels)
        side = config.total_downscale_factor * base_cfg.vae_scale_factor * 2 ** len(base_cfg.block_out_channels)
        check_placements(config, base_cfg, side, side)
        if state_dict is None:
            state_dict = synthetic_t2i_adapter_state_dict(config, seed=zlib.crc32(model_key.encode()) & 0x7FFFFFFF)
        self.cfg, self.base_cfg = config, base_cfg
        self.engine = NativeT2IAdapter(config, state_dict, device)

    def features(self, image: torch.Tensor, scale: float = 1.0) -> List[torch.Tensor]:
        return self.engine.features(image, scale)


class T2IRequest:
    """The T2I-Adapter of one sample() call: its features for the call's batch (B rows each, NHWC fp16) and the
    conditioning factor."""

    def __init__(self, features: Sequence[torch.Tensor], factor: float):
        self.features, self.factor = list(features), float(factor)

    def entry_flags(self, steps) -> List[bool]:
        return entry_flags(steps, self.factor)

    def step_on(self, i: int, n: int) -> bool:
        return step_flags(n, self.factor)[i]


def check_t2i_image(image, cfg: T2IAdapterConfig, batch: int, height: int, width: int) -> torch.Tensor:
    """`image` (B or 1, in_channels, H, W) at exactly the output size (never resized). Returns the (batch, C, H, W)
    tensor. Raises ValueError otherwise."""
    if not torch.is_tensor(image) or image.dim() != 4:
        raise ValueError("t2i_adapter_image must be a (B, C, H, W) tensor")
    if image.shape[1] != cfg.in_channels:
        raise ValueError(f"t2i_adapter_image has {image.shape[1]} channels, the adapter takes {cfg.in_channels}")
    if tuple(image.shape[2:]) != (height, width):
        raise ValueError(f"t2i_adapter_image is {tuple(image.shape[2:])}, the output is {(height, width)}: "
                         "it is not resized, pass it at the output size")
    if image.shape[0] not in (1, batch):
        raise ValueError(f"t2i_adapter_image has {image.shape[0]} images for a batch of {batch}")
    tf = cfg.total_downscale_factor
    if height % tf or width % tf:
        raise ValueError(f"the output size {width}x{height} must be a multiple of the adapter's factor {tf}")
    return image.expand(batch, -1, -1, -1)


def t2i_request(kwargs: dict, unet_cfg: UNetConfig, batch: int, height: int, width: int) -> Optional[T2IRequest]:
    """The T2IRequest of a text-to-image sample() call's keyword arguments (t2i_adapter=, t2i_adapter_image=,
    adapter_conditioning_scale=, adapter_conditioning_factor=), or None without t2i_adapter=. Runs the adapter once.
    Raises ValueError on a missing or mis-sized image, a wrong channel count, a factor outside [0, 1] or an adapter
    whose features do not fit `unet_cfg`."""
    ad, image = kwargs.get("t2i_adapter"), kwargs.get("t2i_adapter_image")
    if ad is None and image is None:
        return None
    if ad is None or image is None:
        raise ValueError("t2i_adapter and t2i_adapter_image go together")
    if not isinstance(ad, T2IAdapter):
        raise ValueError("t2i_adapter= takes a cfgpp_b200.t2i_adapter.T2IAdapter")
    factor = float(kwargs.get("adapter_conditioning_factor", 1.0))
    if not 0.0 <= factor <= 1.0:
        raise ValueError(f"adapter_conditioning_factor must be in [0, 1] (got {factor})")
    image = check_t2i_image(image, ad.cfg, batch, height, width)
    check_placements(ad.cfg, unet_cfg, height, width)
    return T2IRequest(ad.features(image, float(kwargs.get("adapter_conditioning_scale", 1.0))), factor)


__all__ = ["NativeT2IAdapter", "T2IAdapter", "T2IAdapterConfig", "T2IRequest", "check_placements", "check_t2i_image",
           "config_from_diffusers", "entry_flags", "step_flags", "synthetic_t2i_adapter_state_dict",
           "t2i_adapter_config", "t2i_adapter_param_specs", "t2i_request", "unet_placements"]
