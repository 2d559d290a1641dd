"""LoRA on the oracle side: the stated merge rule in fp64, and the unmerged form every LoRA trainer optimises.

Adapters are `{diffusers weight key: (down [r, K], up [N, r], alpha)}` (cfgpp_b200.lora.LoraAdapter.targets has this
form); `scales` has one entry per adapter.

    merge_state_dict: W_eff = fp16( W + sum_a c_a * up_a @ down_a ),  c_a = fp32(fp32(s_a * alpha_a) / r_a)
    attach:           y = base(x) + c_a * up_a(down_a(x))   on Linear and Conv2d (peft's LoRA forward, restated)

The coefficient is formed in fp32 as the engine forms it; everything else is fp64 with one rounding at the end.
peft and diffusers are not installed here, so `attach` is unpinned against them.
"""
from __future__ import annotations

from typing import Dict, Mapping, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

Targets = Mapping[str, Tuple[torch.Tensor, torch.Tensor, float]]


def coef(scale: float, alpha: float, rank: int) -> float:
    return float(np.float32(np.float32(scale) * np.float32(alpha)) / np.float32(rank))


def merged_weight(w: torch.Tensor, factors, dtype=torch.float16) -> torch.Tensor:
    """factors: [(down, up, c)] for one weight; returns the merged weight in `dtype` with w's shape."""
    acc = w.double().reshape(w.shape[0], -1).clone()
    for down, up, c in factors:
        acc += c * (up.double().to(w.device) @ down.double().to(w.device))
    return acc.reshape(w.shape).to(dtype)


def merge_state_dict(sd: Mapping[str, torch.Tensor], adapters: Sequence[Targets], scales: Sequence[float],
                     dtype=torch.float16) -> Dict[str, torch.Tensor]:
    """The expected weights: every targeted key merged by the rule above, the others passed through."""
    per_key: Dict[str, list] = {}
    for targets, s in zip(adapters, scales):
        for key, (down, up, alpha) in targets.items():
            per_key.setdefault(key, []).append((down, up, coef(s, alpha, down.shape[0])))
    return {k: merged_weight(v, per_key[k], dtype) if k in per_key else v for k, v in sd.items()}


class _LoraLayer(nn.Module):
    """base(x) + sum_a c_a * up_a(down_a(x)) around an nn.Linear or nn.Conv2d."""

    def __init__(self, base: nn.Module, factors):
        super().__init__()
        self.base = base
        self.factors = [(d.to(base.weight), u.to(base.weight), c) for d, u, c in factors]

    @property
    def weight(self):
        return self.base.weight

    def forward(self, x):
        y = self.base(x)
        for down, up, c in self.factors:
            if isinstance(self.base, nn.Linear):
                y = y + c * F.linear(F.linear(x, down), up)
            else:
                b = self.base
                r = down.shape[0]
                h = F.conv2d(x, down.reshape(r, *b.weight.shape[1:]), None, b.stride, b.padding)
                y = y + c * F.conv2d(h, up.reshape(up.shape[0], r, 1, 1))
        return y


def attach(unet: nn.Module, adapters: Sequence[Targets], scales: Sequence[float]) -> nn.Module:
    """Wrap, in place, every targeted Linear / Conv2d of an oracle UNet in its unmerged LoRA form."""
    per_key: Dict[str, list] = {}
    for targets, s in zip(adapters, scales):
        for key, (down, up, alpha) in targets.items():
            per_key.setdefault(key, []).append((down, up, coef(s, alpha, down.shape[0])))
    for key, factors in per_key.items():
        path = key[:-len(".weight")].split(".")
        parent = unet
        for p in path[:-1]:
            parent = getattr(parent, p) if not p.isdigit() else parent[int(p)]
        leaf = path[-1]
        base = parent[int(leaf)] if leaf.isdigit() else getattr(parent, leaf)
        assert isinstance(base, (nn.Linear, nn.Conv2d)), f"{key} is not a Linear / Conv2d of the oracle"
        wrapped = _LoraLayer(base, factors)
        if leaf.isdigit():
            parent[int(leaf)] = wrapped
        else:
            setattr(parent, leaf, wrapped)
    return unet
