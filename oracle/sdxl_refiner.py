"""ORACLE (test infrastructure — never imported by the product path).

SDXL 1.0's second expert, the refiner UNet, on top of the existing restatements:

* `sdxl_refiner_config()`: diffusers' UNet2DConditionModel config of stabilityai/stable-diffusion-xl-refiner-1.0 for
  `oracle.unet`, which builds it unchanged: its text_time add-embedding flattens however many time ids it is given
  (here 5: original h, original w, crop top, crop left, aesthetic score; 2560 = 1280 + 5 * 256).
  2,259,526,660 parameters.
* the expert split, applied around the unchanged sampler loops of `oracle.samplers`.

The reference has no refiner, so the split is a stated rule (diffusers' "ensemble of experts": `denoising_end` on
the base pipeline, `denoising_start` on the refiner's), not a restatement:
    k = #{t in timesteps : t >= round(1000 * (1 - denoising_end))}, 0 < denoising_end < 1 and 1 <= k <= n - 1
    (n = number of sampler steps).
    The base UNet, under the base's conditioning, runs steps [0, k) of the one schedule and hands over the sampler
    state itself (zt for the DDIM family, the VE-scaled x for DPM++), not its z0t. The refiner UNet, under its own
    conditioning, runs steps [k, n) of the same schedule and guidance from that state.
    DDIM family (ddim, ddim_cfg++): nothing else changes; the loop is the unsplit loop with the UNet switched at
    call k (`ExpertUNet`).
    dpm++_2m_cfgpp: the refiner starts with no multistep history, as a new diffusers refiner call does: step k
    takes the first-order update (old_denoised = None); every other step is the unsplit loop's
    (`sdxl_dpmpp_2m_cfgpp_split`).
"""
from __future__ import annotations

from typing import Optional

import torch

from .samplers import ddim_plain, predict_noise, sdxl_ddim_cfgpp, sigma_to_t
from .schedule import NUM_TRAIN_TIMESTEPS, ScheduleTables
from .unet import UNetConfig


def sdxl_refiner_config(sample_size: int = 128) -> UNetConfig:
    return UNetConfig(
        name="sdxl_refiner", sample_size=sample_size, block_out_channels=(384, 768, 1536, 1536),
        down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
        up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
        transformer_layers_per_block=(4, 4, 4, 4), num_attention_heads=(6, 12, 24, 24), cross_attention_dim=1280,
        use_linear_projection=True, addition_embed_type="text_time", addition_time_embed_dim=256,
        projection_class_embeddings_input_dim=2560, pooled_dim=1280)


def split_index(timesteps: torch.Tensor, denoising_end: float, nsteps: int) -> int:
    if not 0.0 < denoising_end < 1.0:
        raise ValueError(f"denoising_end {denoising_end} not in (0, 1)")
    k = int((timesteps >= int(round(NUM_TRAIN_TIMESTEPS * (1.0 - denoising_end)))).sum())
    if not 1 <= k <= nsteps - 1:
        raise ValueError(f"split index {k} not in [1, {nsteps - 1}]")
    return k


class ExpertUNet:
    """The two experts seen as the one UNet the loops of `oracle.samplers` call: calls [0, k) go to `base` under
    `base_cond`, the rest to `refiner` under `refiner_cond`, each cond (uc, c, added_cond_kwargs). The conditioning
    the loop passes is replaced by the expert's own."""

    def __init__(self, base, base_cond, refiner, refiner_cond, k: int):
        self.experts = ((base, base_cond), (refiner, refiner_cond))
        self.k, self.calls = k, 0

    def __call__(self, z_in, t, encoder_hidden_states=None, added_cond_kwargs=None):
        unet, (uc, c, add) = self.experts[int(self.calls >= self.k)]
        self.calls += 1
        return unet(z_in, t, encoder_hidden_states=torch.cat([uc, c], dim=0), added_cond_kwargs=add)


@torch.no_grad()
def sdxl_ddim_cfgpp_split(base, refiner, tb: ScheduleTables, zT, base_cond, refiner_cond, cfg_guidance, k,
                          record: Optional[list] = None):
    uc, c, add = base_cond
    return sdxl_ddim_cfgpp(ExpertUNet(base, base_cond, refiner, refiner_cond, k), tb, zT, uc, c, cfg_guidance, add,
                           record=record)


@torch.no_grad()
def sdxl_ddim_split(base, refiner, tb: ScheduleTables, zT, base_cond, refiner_cond, cfg_guidance, k,
                    record: Optional[list] = None):
    uc, c, add = base_cond
    return ddim_plain(ExpertUNet(base, base_cond, refiner, refiner_cond, k), tb, zT, uc, c, cfg_guidance, add,
                      sdxl_indexing=True, record=record)


@torch.no_grad()
def sdxl_dpmpp_2m_cfgpp_split(base, refiner, tb: ScheduleTables, noise, base_cond, refiner_cond, cfg_guidance, k,
                              record: Optional[list] = None):
    """samplers.sdxl_dpmpp_2m_cfgpp with the experts switched at step k and the multistep history dropped there."""
    unet = ExpertUNet(base, base_cond, refiner, refiner_cond, k)
    uc, c, add = base_cond
    alphas = tb.alphas_cumprod[tb.timesteps.int().cpu()].cpu()
    sigmas = (1 - alphas).sqrt() / alphas.sqrt()
    x = noise.to(torch.float16)
    x = x * sigmas[0]
    t_fn = lambda sigma: sigma.log().neg()  # noqa: E731
    old_denoised = None
    for i, _ in enumerate(tb.timesteps[:-1].int()):
        if i == k:
            old_denoised = None
        at = alphas[i]
        sigma = sigmas[i]
        c_in = at.clone().sqrt()
        c_out = -sigma.clone()
        new_t = sigma_to_t(tb, sigma).to(x.device)
        noise_uc, noise_c = predict_noise(unet, x * c_in, new_t, uc, c, add)
        noise_pred = noise_uc + cfg_guidance * (noise_c - noise_uc)
        if record is not None:
            record.append({"x": x.clone(), "noise_uc": noise_uc.clone(), "noise_c": noise_c.clone(),
                           "old_denoised": None if old_denoised is None else old_denoised.clone()})
        denoised = x + c_out * noise_pred
        uncond_denoised = x + c_out * noise_uc
        t, t_next = t_fn(sigmas[i]), t_fn(sigmas[i + 1])
        h = t_next - t
        if old_denoised is None or sigmas[i + 1] == 0:
            x = denoised + (x - uncond_denoised) / sigmas[i].item() * sigmas[i + 1]
        else:
            h_last = t - t_fn(sigmas[i - 1])
            r = h_last / h
            extra1 = -torch.exp(-h) * uncond_denoised - (-h).expm1() * (uncond_denoised - old_denoised) / (2 * r)
            extra2 = torch.exp(-h) * x
            x = denoised + extra1 + extra2
        old_denoised = uncond_denoised
    return x
