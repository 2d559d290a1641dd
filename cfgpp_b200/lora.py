"""LoRA adapters for the UNet: reading the file formats in the wild into factors per diffusers weight key, and the
`load_lora` surface of the solvers. The merge itself runs on the device (csrc/lora.cu) into the engine's packed weights.

For a base weight W viewed as [N, K] (K = every dimension after the first; a 3x3 convolution in its (Cout,Cin,3,3) order)
an adapter holds down [r, K], up [N, r] and alpha, and the engine forms

    W_eff = fp16( fp32(W) + sum_a  s_a * alpha_a / r_a * (up_a @ down_a) )

with fp32 accumulation and one rounding. Factors are held in fp16: an fp32 or bf16 file is rounded once, here.

Three namings are accepted, all resolved through a table built forwards from `weights.unet_param_specs(cfg)`:
  1. diffusers / peft: `[unet.]<module>.lora_A.weight` / `.lora_B.weight`, the older `<module>.lora.down.weight` /
     `.lora.up.weight` and the attention-processor form `...attn1.processor.to_q_lora.down.weight`;
  2. kohya with diffusers module names: `lora_unet_<module with . -> _>.lora_down.weight` / `.lora_up.weight` / `.alpha`;
  3. kohya with the original (SGM / LDM) block numbering (`input_blocks`, `middle_block`, `output_blocks`), which most
     SDXL files use.
The SGM numbering is written from knowledge of the formats: no published LoRA file was available to pin it against.
`alpha` absent means alpha = r (diffusers / peft keep it in a config next to the file: pass `alpha=`).
Text-encoder entries are collected, warned about once and not applied; DoRA, LoHa, LoKr and `lora_mid` are refused.
"""
from __future__ import annotations

import math
import os
import warnings
from dataclasses import dataclass, field
from types import MappingProxyType
from typing import Dict, List, Mapping, Optional, Tuple, Union

import torch

from .config import UNetConfig
from .weights import unet_param_specs

MAX_RANK = 128
NAMINGS = ("diffusers", "kohya", "kohya_sgm")
_RESNET_SGM = {"norm1": "in_layers.0", "conv1": "in_layers.2", "time_emb_proj": "emb_layers.1", "norm2": "out_layers.0",
               "conv2": "out_layers.3", "conv_shortcut": "skip_connection"}
# (suffix, role), longest first so that `_lora.down.weight` is not read as `.down.weight` of something else
_SUFFIXES = ((".lora_A.weight", "down"), (".lora_B.weight", "up"), (".lora.down.weight", "down"),
             (".lora.up.weight", "up"), ("_lora.down.weight", "down"), ("_lora.up.weight", "up"),
             (".lora_down.weight", "down"), (".lora_up.weight", "up"), (".alpha", "alpha"))
_REFUSED = (("dora_scale", "DoRA"), ("hada_", "LoHa"), ("lokr_", "LoKr"), ("lora_mid", "a Tucker-decomposed conv LoRA"))


@dataclass
class LoraAdapter:
    """targets: diffusers weight key -> (down [r, K] fp16, up [N, r] fp16, alpha)."""
    targets: Dict[str, Tuple[torch.Tensor, torch.Tensor, float]]
    skipped_text_encoder: List[str] = field(default_factory=list)
    name: Optional[str] = None


def sgm_module(module: str, cfg: UNetConfig) -> str:
    """The original (SGM / LDM) name of a diffusers UNet module."""
    p = module.split(".")
    n = cfg.layers_per_block + 1
    top = {"conv_in": "input_blocks.0.0", "conv_norm_out": "out.0", "conv_out": "out.2"}
    if p[0] in top:
        return top[p[0]]
    if p[0] == "time_embedding":
        return f"time_embed.{0 if p[1] == 'linear_1' else 2}"
    if p[0] == "add_embedding":
        return f"label_emb.0.{0 if p[1] == 'linear_1' else 2}"

    def inner(kind, rest):
        return ".".join([_RESNET_SGM[rest[0]]] + rest[1:]) if kind == "resnets" else ".".join(rest)

    if p[0] == "mid_block":
        slot = {("resnets", "0"): 0, ("attentions", "0"): 1, ("resnets", "1"): 2}[(p[1], p[2])]
        return f"middle_block.{slot}." + inner(p[1], p[3:])
    i, kind, j = int(p[1]), p[2], int(p[3])
    if p[0] == "down_blocks":
        if kind == "downsamplers":
            return f"input_blocks.{(i + 1) * n}.0.op"
        return f"input_blocks.{1 + i * n + j}.{0 if kind == 'resnets' else 1}." + inner(kind, p[4:])
    assert p[0] == "up_blocks", module
    if kind == "upsamplers":
        has_attn = cfg.up_block_types[i] == "CrossAttnUpBlock2D"
        return f"output_blocks.{i * n + n - 1}.{2 if has_attn else 1}.conv"
    return f"output_blocks.{i * n + j}.{0 if kind == 'resnets' else 1}." + inner(kind, p[4:])


def module_spellings(cfg: UNetConfig) -> Dict[str, Dict[str, str]]:
    """diffusers weight key -> {naming: the module stem a file of that naming uses}, for every parameter of two or more
    dimensions (the ones an adapter can target)."""
    out = {}
    for key, shape, _ in unet_param_specs(cfg):
        if len(shape) < 2:
            continue
        module = key[:-len(".weight")]
        out[key] = {"diffusers": module, "kohya": "lora_unet_" + module.replace(".", "_"),
                    "kohya_sgm": "lora_unet_" + sgm_module(module, cfg).replace(".", "_")}
    return out


def _stem_table(cfg: UNetConfig) -> Dict[str, str]:
    table = {}
    for key, sp in module_spellings(cfg).items():
        for stem in sp.values():
            table[stem] = key
        head, _, leaf = sp["diffusers"].rpartition(".")
        if head.endswith((".attn1", ".attn2")):  # attention-processor form: attn1.processor.to_q_lora / to_out_lora
            table[f"{head}.processor.{leaf}"] = key
        elif head.endswith(".to_out"):
            table[f"{head[:-len('.to_out')]}.processor.to_out"] = key
    return table


def is_lora_keys(keys) -> bool:
    """Whether a state dict's keys are those of a LoRA file rather than of a full UNet."""
    return any(k.endswith(s) for k in keys for s, role in _SUFFIXES if role != "alpha")


def is_lora_file(path: str) -> bool:
    from safetensors import safe_open
    with safe_open(path, framework="pt") as f:
        return is_lora_keys(list(f.keys()))


def read_lora(path_or_dict: Union[str, os.PathLike, Mapping[str, torch.Tensor]], cfg: UNetConfig,
              alpha: Optional[float] = None) -> LoraAdapter:
    """Read a LoRA state dict (or `*.safetensors` file) for the UNet `cfg` describes. `alpha`: the value for targets the
    file gives none (default: each target's rank). Factors of any float dtype are rounded once to fp16. Raises
    ValueError naming the key for an unsupported variant, a rank above 128, a shape that does not fit the base weight or
    a key that maps to no UNet weight."""
    name = None
    if not isinstance(path_or_dict, Mapping):
        from safetensors.torch import load_file
        name = os.path.splitext(os.path.basename(os.fspath(path_or_dict)))[0]
        path_or_dict = load_file(os.fspath(path_or_dict))
    table = _stem_table(cfg)
    shapes = {k: s for k, s, _ in unet_param_specs(cfg)}
    parts: Dict[str, Dict[str, torch.Tensor]] = {}
    skipped: List[str] = []
    for fk, t in path_or_dict.items():
        for marker, what in _REFUSED:
            if marker in fk:
                raise ValueError(f"LoRA key '{fk}': {what} is not supported")
        stem = fk[len("unet."):] if fk.startswith("unet.") else fk
        if stem.startswith(("lora_te", "text_encoder")):
            skipped.append(fk)
            continue
        for suffix, role in _SUFFIXES:
            if stem.endswith(suffix):
                stem = stem[:-len(suffix)]
                break
        else:
            raise ValueError(f"LoRA key '{fk}' is not a LoRA factor or alpha")
        if stem not in table:
            raise ValueError(f"LoRA key '{fk}' maps to no weight of the {cfg.name} UNet")
        parts.setdefault(table[stem], {})[role] = t
        parts[table[stem]][role + "_key"] = fk
    if skipped:
        warnings.warn(f"{len(skipped)} text-encoder LoRA tensors are not applied (UNet adapters only)")
    targets = {}
    for key, p in parts.items():
        if "down" not in p or "up" not in p:
            raise ValueError(f"LoRA target '{key}' lacks its {'down' if 'down' not in p else 'up'} factor")
        down, up = p["down"], p["up"]
        if up.dim() == 4 and tuple(up.shape[2:]) != (1, 1):
            raise ValueError(f"LoRA key '{p['up_key']}': an up factor with a {up.shape[2]}x{up.shape[3]} kernel is not supported")
        r = down.shape[0]
        if r > MAX_RANK:
            raise ValueError(f"LoRA key '{p['down_key']}': rank {r} exceeds {MAX_RANK}")
        N, K = shapes[key][0], math.prod(shapes[key][1:])
        down, up = down.reshape(r, -1), up.reshape(up.shape[0], -1)
        if tuple(down.shape) != (r, K) or tuple(up.shape) != (N, r):
            raise ValueError(f"LoRA key '{p['down_key']}': factors {tuple(p['down'].shape)} / {tuple(p['up'].shape)} do "
                             f"not fit the base weight {key} {tuple(shapes[key])}")
        a = float(p["alpha"]) if "alpha" in p else (float(r) if alpha is None else float(alpha))
        targets[key] = (down.to(torch.float16).contiguous(), up.to(torch.float16).contiguous(), a)
    return LoraAdapter(targets, skipped, name)


class LoraMixin:
    """`load_lora` surface of the solvers and of SDXLRefiner (anything with `.unet`, a NativeUNet, and `.cfg`)."""

    def load_lora(self, path_or_dict, scale: float = 1.0, name: Optional[str] = None) -> str:
        """Merge a LoRA (file or state dict, see read_lora) into this solver's UNet at `scale`; returns its name.
        Adapters are state of the ENGINE, and solvers built with the same `model_key` share one engine: every one of
        them runs with the adapter from now on (`loras` of each shows it). Switching scale or adapter re-merges on the
        device from a pristine copy of the weights; the plan and the captured graph are kept."""
        adapter = path_or_dict if isinstance(path_or_dict, LoraAdapter) else read_lora(path_or_dict, self.cfg)
        return self.unet.add_lora(adapter, scale, name or adapter.name)

    def set_lora_scale(self, name: str, scale: float) -> None:
        self.unet.set_lora_scales({name: scale})

    def unload_lora(self) -> None:
        """Remove every adapter: the base weights bit for bit, backups freed."""
        self.unet.clear_lora()

    @property
    def loras(self) -> Mapping[str, float]:
        """name -> scale of the adapters the engine this solver runs on carries (read-only)."""
        return MappingProxyType(dict(self.unet.loras))
