"""k-diffusion (VE-cast) samplers on the native UNet seam — CFG++ variants (SURVEY §8 f1) and, with `cfgpp=False`, the
plain-CFG baselines they are compared against (§8 f4: latent_diffusion.py:302-503, latent_sdxl.py:469-517).

The reference expresses `euler_cfg++`, `euler_a_cfg++`, `dpm++_2s_a_cfg++` and `dpm++_2m_cfg++` through one helper,
`kdiffusion_x_to_denoised` (latent_diffusion.py:232-241; SDXL twin `kdiffusion_zt_to_denoised`, latent_sdxl.py:357-363):
scale the VE state to the VP input, ONE batched uncond+cond UNet call through `predict_noise`, CFG mix, two Tweedie
estimates (guided and unconditional). CFG++ then renoises / extrapolates with the UNCONDITIONAL estimate. Here the UNet
call is the Blackwell-native forward (`cfgpp_unet_forward` behind `predict_noise`); the per-step sampler arithmetic of
these variants is a handful of elementwise fp16 tensor ops and stays in torch — >99.9 % of a step is the UNet. Their
fused-epilogue versions (as done for ddim_cfg++ / dpm++_2m_cfgpp) are a later optimisation, not a semantic change.

dtype behaviour mirrored from the reference: the state `x` is fp16; `sigmas` is a CPU fp32 table whose 0-dim entries
enter CUDA tensor ops as fp32 scalars (the result stays fp16); `to_d` divides by a Python float (`sigma.item()`).
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence

import torch

from . import schedule as S
from .batching import guidance_mix, guidance_table


def get_ancestral_step(sigma_from, sigma_to, eta: float = 1.):
    """(sigma_down, sigma_up) of an ancestral step — latent_diffusion.py:30-37."""
    if not eta:
        return sigma_to, 0.
    var_ratio = sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2
    sigma_up = min(sigma_to, eta * var_ratio ** 0.5)
    return (sigma_to ** 2 - sigma_up ** 2) ** 0.5, sigma_up


def append_zero(x: torch.Tensor) -> torch.Tensor:
    return torch.cat([x, x.new_zeros([1])])


def get_sigmas_karras(n: int, sigma_min, sigma_max, rho: float = 7., device='cpu') -> torch.Tensor:
    """Karras et al. (2022) noise levels, n values + a trailing 0 — latent_diffusion.py:44-50."""
    ramp = torch.linspace(0, 1, n + 1, device=device)[:-1]
    lo, hi = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    return append_zero((hi + ramp * (lo - hi)) ** rho).to(device)


class KDiffusionMixin:
    """Methods the k-diffusion samplers call on the solver object (latent_diffusion.py:211-241, latent_sdxl.py:341-363).
    The host class provides `predict_noise`, `log_sigmas`, `total_alphas`, `device`."""

    def timestep(self, sigma: torch.Tensor) -> torch.Tensor:
        """Index of the training noise level nearest to sigma in log space."""
        dists = sigma.log().to(self.log_sigmas.device) - self.log_sigmas[:, None]
        return dists.abs().argmin(dim=0).view(sigma.shape).to(sigma.device)

    def to_d(self, x, sigma, denoised):
        """Karras ODE derivative of a denoiser output."""
        return (x - denoised) / sigma.item()

    def calculate_input(self, x, sigma):
        return x / (sigma ** 2 + 1) ** 0.5

    def calculate_denoised(self, x, model_pred, sigma):
        return x - model_pred * sigma

    def total_sigmas(self) -> torch.Tensor:
        return (1 - self.total_alphas).sqrt() / self.total_alphas.sqrt()

    def _k_denoise(self, x, sigma, t, cfg_guidance, cond: Sequence):
        """cond = (uc, c) for SD v1.5, (uc, c, add_cond_kwargs) for SDXL. Returns (denoised, uncond_denoised)."""
        xc = self.calculate_input(x, sigma)
        if getattr(self, "v_prediction", False):
            # v -> eps at the level the VE update assigns to x (abar = 1 / (1 + sigma^2)), as the fused step does
            v_uc, v_c = self.model_output(xc, t, *cond)
            a, b = S.ve_v_coefs(sigma)
            noise_uc, noise_c = S.v_to_eps(v_uc, xc, a, b), S.v_to_eps(v_c, xc, a, b)
        else:
            noise_uc, noise_c = self.predict_noise(xc, t, *cond)
        noise_pred = guidance_mix(noise_uc, noise_c, cfg_guidance)
        return self.calculate_denoised(x, noise_pred, sigma), self.calculate_denoised(x, noise_uc, sigma)

    def kdiffusion_x_to_denoised(self, x, sigma, uc, c, cfg_guidance, t):
        return self._k_denoise(x, sigma, t, cfg_guidance, (uc, c))

    def kdiffusion_zt_to_denoised(self, x, sigma, uc, c, cfg_guidance, t, add_cond_kwargs):
        return self._k_denoise(x, sigma, t, cfg_guidance, (uc, c, add_cond_kwargs))


def _fused_trajectory(solver, x, steps, cond, cfg_guidance, noise_slots: int = 0):
    """Whole VE-cast trajectory on the fused step kernel (UNet + CFG / CFG++ mix + Euler / DPM++2M update in the conv_out
    epilogue, one CUDA-graph replay per step, no elementwise launch or host sync in between). Returns (last denoised, x).
    Ancestral loops (`noise_slots` > 0, see schedule.kd_ancestral_steps): the fresh noise of every step is drawn up
    front, in loop order, with the calls the op-by-op loop would make (`torch.randn_like(x)`, same generator state =>
    same values), and travels as a table the step kernel indexes; dpm++_2s_a replays the graph twice per step
    (midpoint, final)."""
    solver._prepare(x, *cond, force=True)
    x = x.to(solver.unet.device, torch.float16)
    noise = torch.stack([torch.randn_like(x) for _ in range(noise_slots)]) if noise_slots else None
    return solver.unet.run_trajectory(S.STEP_DPMPP2M_CFGPP, torch.float16, steps, x, guidance_table(cfg_guidance),
                                      noise, solver._control_entries(steps))


def _control_step(solver, i: int, n: int) -> None:
    """The ControlNet scale of step i of n before its UNet call(s) (solvers without one have no hook)."""
    hook = getattr(solver, "_control_step", None)
    if hook is not None:
        hook(i, n)


def _fusable(solver, callback_fn) -> bool:
    """Deterministic loops without a callback run fused when the solver sits on the native engine (the CPU tests drive
    these loops with a stand-in UNet and keep the op-by-op torch form, which stays the specification)."""
    from .engine import NativeUNet
    return callback_fn is None and isinstance(getattr(solver, "unet", None), NativeUNet)


def _callback(callback_fn: Optional[Callable], i, t, z0t, zt, decode):
    if callback_fn is None:
        return z0t, zt
    kw = callback_fn(i, t, {'z0t': z0t.detach(), 'zt': zt.detach(), 'decode': decode})
    return kw["z0t"], kw["zt"]


@torch.no_grad()
def euler_cfgpp_loop(solver: KDiffusionMixin, x, sigmas, cfg_guidance, cond, callback_fn=None,
                     ancestral: bool = False, adopt_callback: bool = True, cfgpp: bool = True):
    """Euler (optionally ancestral) CFG++: x' = D_guided(x) + sigma' * (x - D_uncond(x)) / sigma  [+ sigma_up * N(0,1)].
    latent_diffusion.py:699-719 (euler_cfg++), :744-762 (euler_a_cfg++), latent_sdxl.py:787-808 (SDXL euler_cfg++).
    Returns (last denoised, x). `adopt_callback`: the ancestral variant of the reference ignores what the callback
    returns (:757-762). `cfgpp=False`: plain CFG, the derivative uses the guided estimate (:326-330, :372-379)."""
    if _fusable(solver, callback_fn):
        if ancestral:
            steps, slots = S.kd_ancestral_steps(sigmas, solver.timestep, cfg_guidance, cfgpp)
            return _fused_trajectory(solver, x, steps, cond, cfg_guidance, slots)
        return _fused_trajectory(solver, x, S.kd_steps(sigmas, solver.timestep, cfg_guidance, cfgpp), cond,
                                 cfg_guidance)
    denoised = None
    for i in range(len(sigmas) - 1):
        sigma = sigmas[i]
        t = solver.timestep(sigma).to(solver.device)
        _control_step(solver, i, len(sigmas) - 1)
        denoised, uncond_denoised = solver._k_denoise(x, sigma, t, cfg_guidance, cond)
        d = solver.to_d(x, sigma, uncond_denoised if cfgpp else denoised)
        if ancestral:
            sigma_down, sigma_up = get_ancestral_step(sigmas[i], sigmas[i + 1])
            x = denoised + d * sigma_down
            if sigmas[i + 1] > 0:
                x = x + torch.randn_like(x) * sigma_up
        else:
            x = denoised + d * sigmas[i + 1]
        z0t, zt = _callback(callback_fn, i, t, denoised, x, solver.decode)
        if adopt_callback and callback_fn is not None:
            denoised, x = z0t, zt
    return denoised, x


@torch.no_grad()
def dpmpp_2s_a_cfgpp_loop(solver: KDiffusionMixin, x, sigmas, cfg_guidance, cond, callback_fn=None,
                          cfgpp: bool = True):
    """DPM-Solver++(2S) ancestral, CFG++: both the midpoint and the final update extrapolate with the unconditional
    Tweedie estimate — latent_diffusion.py:782-825 (two UNet calls per step). `cfgpp=False`: the plain-CFG original
    (:408-437), guided estimate everywhere and the standard final update."""
    if _fusable(solver, callback_fn):
        steps, slots = S.kd_ancestral_steps(sigmas, solver.timestep, cfg_guidance, cfgpp, two_s=True)
        return _fused_trajectory(solver, x, steps, cond, cfg_guidance, slots)
    t_fn = lambda s: s.log().neg()      # noqa: E731
    sigma_fn = lambda t: t.neg().exp()  # noqa: E731
    denoised = None
    for i in range(len(sigmas) - 1):
        sigma = sigmas[i]
        new_t = solver.timestep(sigma).to(solver.device)
        _control_step(solver, i, len(sigmas) - 1)  # both UNet calls of the step take its scale
        denoised, uncond_denoised = solver._k_denoise(x, sigma, new_t, cfg_guidance, cond)
        sigma_down, sigma_up = get_ancestral_step(sigmas[i], sigmas[i + 1])
        extrap = uncond_denoised if cfgpp else denoised
        if sigma_down == 0:
            x = denoised + solver.to_d(x, sigmas[i], extrap) * sigma_down
        else:
            t, t_next = t_fn(sigmas[i]), t_fn(sigma_down)
            r = 1 / 2
            h = t_next - t
            s = t + r * h
            x_2 = (sigma_fn(s) / sigma_fn(t)) * x - (-h * r).expm1() * extrap
            sigma_s = sigma_fn(s)
            t_2 = solver.timestep(sigma_s).to(solver.device)
            denoised_2, uncond_denoised_2 = solver._k_denoise(x_2, sigma_s, t_2, cfg_guidance, cond)
            if cfgpp:
                x = denoised_2 - torch.exp(-h) * uncond_denoised_2 + (sigma_fn(t_next) / sigma_fn(t)) * x
            else:
                x = (sigma_fn(t_next) / sigma_fn(t)) * x - (-h).expm1() * denoised_2
        if sigmas[i + 1] > 0:
            x = x + torch.randn_like(x) * sigma_up
        denoised, x = _callback(callback_fn, i, new_t, denoised, x, solver.decode)
    return denoised, x


@torch.no_grad()
def dpmpp_2m_cfgpp_karras_loop(solver: KDiffusionMixin, x, sigmas, cfg_guidance, cond, callback_fn=None,
                               cfgpp: bool = True):
    """SD v1.5 `dpm++_2m_cfg++` (latent_diffusion.py:847-877). NOTE the reference's two files differ: this variant's
    second-order term uses (denoised - old_denoised) with the GUIDED estimate, SDXL's `dpm++_2m_cfgpp` uses the
    unconditional one (latent_sdxl.py:916; that one runs on the fused step kernel). `cfgpp=False`: plain `dpm++_2m`
    (:470-487), guided estimate everywhere."""
    if _fusable(solver, callback_fn):
        return _fused_trajectory(solver, x, S.kd_steps(sigmas, solver.timestep, cfg_guidance, cfgpp, second_order=True,
                                                       diff_guided=True), cond, cfg_guidance)
    t_fn = lambda s: s.log().neg()  # noqa: E731
    old_denoised = None
    denoised = None
    for i in range(len(sigmas) - 1):
        sigma = sigmas[i]
        new_t = solver.timestep(sigma).to(solver.device)
        _control_step(solver, i, len(sigmas) - 1)
        denoised, uncond_denoised = solver._k_denoise(x, sigma, new_t, cfg_guidance, cond)
        t, t_next = t_fn(sigmas[i]), t_fn(sigmas[i + 1])
        h = t_next - t
        extrap = uncond_denoised if cfgpp else denoised
        if old_denoised is None or sigmas[i + 1] == 0:
            x = denoised + solver.to_d(x, sigmas[i], extrap) * sigmas[i + 1]
        else:
            h_last = t - t_fn(sigmas[i - 1])
            r = h_last / h
            extra1 = -torch.exp(-h) * extrap - (-h).expm1() * (denoised - old_denoised) / (2 * r)
            extra2 = torch.exp(-h) * x
            x = denoised + extra1 + extra2
        old_denoised = extrap
        denoised, x = _callback(callback_fn, i, new_t, denoised, x, solver.decode)
    return denoised, x
