"""Argument handling of batched `sample()` calls: many prompts per trajectory, one guidance scale per image.

The reference's solvers take one prompt (latent_sdxl.py:96-99 notes batch_size = 1 as a limitation). Here
`prompt[1]` may be a list of B strings, the null prompt one string (broadcast) or B strings, `cfg_guidance` a float or
B floats, and `zT` a (B,4,h,w) draw; the solver runs all B images as one trajectory (UNet batch 2B). A sequence of
guidance scales reaches the fused step kernel as a per-image table (`cfgpp_set_guidance`); the step table keeps a
scalar. A sequence whose entries are all equal is the scalar call, bit for bit.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

Guidance = Union[float, Sequence[float]]


def _is_seq(x) -> bool:
    return isinstance(x, (list, tuple))


def guidance_table(cfg_guidance: Guidance) -> Optional[List[float]]:
    """The per-image guidance table, or None for a scalar guidance scale."""
    return [float(g) for g in cfg_guidance] if _is_seq(cfg_guidance) else None


def guidance_values(cfg_guidance: Guidance) -> List[float]:
    return guidance_table(cfg_guidance) or [float(cfg_guidance)]


def schedule_lambda(cfg_guidance: Guidance) -> float:
    """The scalar the step table carries: the guidance scale itself, or the first image's entry when a per-image table
    overrides it."""
    return guidance_values(cfg_guidance)[0]


def guidance_mix(noise_uc: torch.Tensor, noise_c: torch.Tensor, cfg_guidance: Guidance) -> torch.Tensor:
    """noise_uc + lambda * (noise_c - noise_uc). A per-image table is applied row by row with Python floats, so every row
    rounds exactly as the scalar call with that row's lambda does."""
    table = guidance_table(cfg_guidance)
    if table is None:
        return noise_uc + cfg_guidance * (noise_c - noise_uc)
    if len(table) != noise_uc.shape[0]:
        raise ValueError(f"{len(table)} guidance scales for a batch of {noise_uc.shape[0]}")
    return torch.cat([noise_uc[b:b + 1] + lam * (noise_c[b:b + 1] - noise_uc[b:b + 1]) for b, lam in enumerate(table)])


def normalize_batch(prompts: Dict[str, Union[str, Sequence[str]]], cfg_guidance: Guidance,
                    zT: Optional[torch.Tensor] = None) -> Tuple[int, Dict[str, Union[str, List[str]]], Guidance]:
    """Batch size B and the normalised arguments of one `sample()` call.

    `prompts` maps argument names to one string or a list of strings; lists must all have length B, strings are
    broadcast. `cfg_guidance` is a float or B floats; `zT` (may be None) must have B rows. B is the common length of
    everything given as a batch (1 if nothing is). Returns (B, prompts with lists as lists, guidance), where a guidance
    sequence whose entries are all equal comes back as that float. Raises ValueError on any length mismatch."""
    sizes = {}
    out = {}
    for name, p in prompts.items():
        if _is_seq(p):
            if not all(isinstance(s, str) for s in p):
                raise ValueError(f"{name} must be a string or a list of strings")
            sizes[name] = len(p)
            out[name] = list(p)
        elif isinstance(p, str):
            out[name] = p
        else:
            raise ValueError(f"{name} must be a string or a list of strings, not {type(p).__name__}")
    table = guidance_table(cfg_guidance)
    if table is not None:
        sizes["cfg_guidance"] = len(table)
    if zT is not None:
        if zT.dim() != 4:
            raise ValueError(f"zT must be (B, 4, h, w), got shape {tuple(zT.shape)}")
        sizes["zT"] = zT.shape[0]
    if any(n == 0 for n in sizes.values()):
        raise ValueError("empty batch: " + ", ".join(k for k, n in sizes.items() if n == 0))
    if len(set(sizes.values())) > 1:
        raise ValueError("batch sizes differ: " + ", ".join(f"{k}={n}" for k, n in sizes.items()))
    B = next(iter(sizes.values()), 1)
    if table is not None and all(g == table[0] for g in table):
        cfg_guidance = table[0]
    elif table is not None:
        cfg_guidance = table
    return B, out, cfg_guidance


def encode_prompts(encode, prompt: Union[str, Sequence[str]], batch: int, takes_list: bool = False):
    """Run `encode(p) -> (hidden, pooled or None)` over one prompt (broadcast to `batch` rows) or a list of prompts.
    `takes_list`: the encoder accepts a list and encodes it in one call (ClipConditioner); otherwise it runs once per
    prompt."""
    if isinstance(prompt, str):
        hidden, pooled = encode(prompt)
        if batch > 1:
            hidden = hidden.expand(batch, *hidden.shape[1:])
            pooled = None if pooled is None else pooled.expand(batch, *pooled.shape[1:])
        return hidden, pooled
    if takes_list:
        return encode(list(prompt))
    outs = [encode(p) for p in prompt]
    hidden = torch.cat([h for h, _ in outs])
    pooled = None if outs[0][1] is None else torch.cat([p for _, p in outs])
    return hidden, pooled


def draw_latents(shape: Sequence[int]) -> torch.Tensor:
    """torch.randn(shape) from the CPU generator, one image at a time in order: image i of a batch is the draw a
    single-image call at the same generator position would make, whatever the batch size."""
    one = (1, *shape[1:])
    return torch.cat([torch.randn(one) for _ in range(shape[0])])


def sdxl_added_conditions(pool_null: torch.Tensor, pool_prompt: torch.Tensor, negative_time_ids: torch.Tensor,
                          time_ids: torch.Tensor, cfg_guidance: Guidance, batch: int):
    """(text_embeds, time_ids) of the SDXL add-embedding for a batch of `batch` images.

    Scalar guidance follows the reference (latent_sdxl.py:249-257): for lambda in {0, 1} the positive pooled embedding
    and time ids are not duplicated (batch rows, broadcast over both CFG halves); otherwise the uncond half gets the
    negative ones (2 * batch rows). With a per-image table every image decides for itself: its uncond row gets the
    positive or the negative embedding by the same rule on its own lambda (always 2 * batch rows)."""
    pos_t = time_ids.reshape(1, -1).expand(batch, -1)
    neg_t = negative_time_ids.reshape(1, -1).expand(batch, -1)
    table = guidance_table(cfg_guidance)
    if table is None:
        if cfg_guidance != 0.0 and cfg_guidance != 1.0:
            return torch.cat([pool_null, pool_prompt], dim=0), torch.cat([neg_t, pos_t], dim=0)
        return pool_prompt, pos_t.contiguous()
    undup = torch.tensor([g == 0.0 or g == 1.0 for g in table], device=pool_prompt.device)
    uc_pool = torch.where(undup[:, None], pool_prompt, pool_null.to(pool_prompt.device))
    uc_t = torch.where(undup.to(pos_t.device)[:, None], pos_t, neg_t)
    return torch.cat([uc_pool, pool_prompt], dim=0), torch.cat([uc_t, pos_t], dim=0)
