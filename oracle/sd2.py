"""ORACLE (test infrastructure — never imported by the product path).

Stable Diffusion 2.x on top of the existing restatements, which need nothing else:

* `sd2_config()` / `sd2_base_config()`: diffusers' UNet2DConditionModel config of stabilityai/stable-diffusion-2-1
  (768^2, v-prediction) and -2-base (512^2, epsilon) for `oracle.unet` — the same network, 865,910,724 parameters.
* the v-prediction rule, applied around the unchanged sampler loops of `oracle.samplers` by `VPredUNet`.

`upcast_attention`: the SD 2.1 unet/config.json sets it to true. In diffusers 0.27.1 the flag only reaches
`Attention.upcast_attention`, which `get_attention_scores` reads — the path of the legacy `AttnProcessor`. The processor
the reference actually runs is the default `AttnProcessor2_0` (torch >= 2), which calls F.scaled_dot_product_attention on
the fp16 q / k / v and never reads the flag. So the oracle takes the same SDPA path as for every other model
(`oracle.unet.Attention.forward`), and the config has no such field.

v-prediction (SD 2.0-v / 2.1). The reference has no v path, so this is a stated rule rather than a restatement:
    eps = fp32(a * v) + fp32(b * x_in), cast back to the model output's dtype (fp16 under autocast),
two products and a sum in fp32 (fp64 when v is fp64), x_in the UNet input as the first conv sees it (z_in cast to the
output dtype), a = sqrt(abar), b = sqrt(1 - abar) with abar the noise level the SAMPLER'S OWN UPDATE assigns to the
state it fed:
    DDIM sampling (ddim, ddim_cfg++ and the sampling half of the edit loops): abar = alpha(t) of the loop
    DDIM inversion: abar = alpha(t - skip) (at_prev: the level of the state being inverted)
    VE-cast loops (euler*, dpm++_2s_a*, dpm++_2m*): abar = 1 / (1 + sigma^2), i.e. a = c_in = 1 / sqrt(sigma^2 + 1)
      and b = sigma * c_in — k-diffusion's VDenoiser; each UNet call of a 2S step with its own sigma.
`VPredUNet` is told the (a, b) of each UNet call in the loop's call order by one of the *_v_levels functions.
"""
from __future__ import annotations

import torch

from .samplers import _alpha_sd15, ancestral_step
from .schedule import ScheduleTables
from .unet import UNetConfig


def sd2_config(sample_size: int = 96) -> UNetConfig:
    """stabilityai/stable-diffusion-2-1: SD v1.5's 4 levels with linear projections, 64-wide heads (diffusers'
    `attention_head_dim` (5, 10, 20, 20)), OpenCLIP ViT-H context (1024)."""
    return UNetConfig(name="sd2", sample_size=sample_size, num_attention_heads=(5, 10, 20, 20),
                      cross_attention_dim=1024, use_linear_projection=True)


def sd2_base_config() -> UNetConfig:
    return sd2_config(sample_size=64)


def v_to_eps(v, x_in, a, b):
    wd = torch.promote_types(v.dtype, torch.float32)
    a = torch.as_tensor(a, dtype=wd)
    b = torch.as_tensor(b, dtype=wd)
    return (v.to(wd) * a.to(v.device) + x_in.to(v.dtype).to(wd) * b.to(v.device)).to(v.dtype)


def ddim_v_levels(tb: ScheduleTables):
    """(a, b) of the sampling loops' calls (descending t): abar = alpha(t)."""
    return [(_alpha_sd15(tb, t).sqrt(), (1 - _alpha_sd15(tb, t)).sqrt()) for t in tb.timesteps]


def inversion_v_levels(tb: ScheduleTables):
    """(a, b) of the inversion loops' calls (ascending t): abar = alpha(t - skip)."""
    out = []
    for t in reversed(tb.timesteps):
        ap = _alpha_sd15(tb, t - tb.skip)
        out.append((ap.sqrt(), (1 - ap).sqrt()))
    return out


def ve_v_level(sigma):
    c_in = torch.tensor(1.0, dtype=torch.float32) / (sigma ** 2 + 1) ** 0.5
    return c_in, sigma * c_in


def kd_v_levels(sigmas, two_s: bool = False):
    """(a, b) of the VE-cast loops' calls: one per sigma_i (i < n); with two_s, the midpoint call at sigma_s follows
    every step whose sigma_down > 0 (samplers.kd_dpmpp_2s_a_cfgpp)."""
    t_fn = lambda sigma: sigma.log().neg()  # noqa: E731
    sigma_fn = lambda t: t.neg().exp()      # noqa: E731
    out = []
    for i in range(len(sigmas) - 1):
        out.append(ve_v_level(sigmas[i]))
        if two_s:
            sigma_down, _ = ancestral_step(sigmas[i], sigmas[i + 1])
            if sigma_down != 0:
                t, t_next = t_fn(sigmas[i]), t_fn(sigma_down)
                out.append(ve_v_level(sigma_fn(t + 0.5 * (t_next - t))))
    return out


class VPredUNet:
    """A v-prediction UNet seen as the eps model the loops of `oracle.samplers` expect: call k converts with
    levels[k]."""

    def __init__(self, unet, levels):
        self.unet, self.levels, self.calls = unet, list(levels), 0

    def __call__(self, z_in, t, encoder_hidden_states=None, added_cond_kwargs=None):
        a, b = self.levels[self.calls]
        self.calls += 1
        v = self.unet(z_in, t, encoder_hidden_states=encoder_hidden_states, added_cond_kwargs=added_cond_kwargs)["sample"]
        return {"sample": v_to_eps(v, z_in, a, b)}
