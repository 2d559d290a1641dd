"""Scheduler tables and per-step scalar coefficients of the CFG++ solvers (product side).

The reference only uses diffusers schedulers as a *table source* (`scheduler.step()` is never called):
  StableDiffusion.__init__   latent_diffusion.py:69-80      SDXL.__init__  latent_sdxl.py:56-67
  SDXLLightning.__init__     latent_sdxl.py:407-418
and computes every per-step scalar with fp32 torch CPU ops inside the loops
  ddim_cfg++ (SD1.5)  latent_diffusion.py:655-656   ddim_cfg++ (SDXL)  latent_sdxl.py:731-734
  inversion           latent_diffusion.py:899-900   dpm++_2m_cfgpp     latent_sdxl.py:877-879, 892-918.
Here the same fp32 torch CPU ops are evaluated once per trajectory into a table (`cfgpp_step_state[]`) that the
fused step kernel indexes on the device — removing the 2–3 host syncs per step the reference incurs
(`alphas_cumprod[t]` indexes a CPU tensor with a CUDA scalar; `t >= 0`).
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

from .batching import schedule_lambda

NUM_TRAIN_TIMESTEPS = 1000

STEP_NONE, STEP_DDIM_CFGPP, STEP_DDIM_INV_CFGPP, STEP_DPMPP2M_CFGPP, STEP_DDIM_CFG = 0, 1, 2, 3, 4
F16, F32 = 0, 1


class StepCoefC(ctypes.Structure):
    _fields_ = [("lambda_", ctypes.c_float), ("c0", ctypes.c_float), ("c1", ctypes.c_float), ("c2", ctypes.c_float),
                ("c3", ctypes.c_float), ("d0", ctypes.c_float), ("d1", ctypes.c_float), ("d2", ctypes.c_float),
                ("d3", ctypes.c_float), ("second_order", ctypes.c_int)]


class StepStateC(ctypes.Structure):
    _fields_ = [("t", ctypes.c_float), ("in_scale", ctypes.c_float), ("coef", StepCoefC)]


def alphas_cumprod_table() -> torch.Tensor:
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, NUM_TRAIN_TIMESTEPS, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def ddim_leading_timesteps(n: int, steps_offset: int = 1) -> torch.Tensor:
    ratio = NUM_TRAIN_TIMESTEPS // n
    ts = (np.arange(0, n) * ratio).round()[::-1].copy().astype(np.int64)
    return torch.from_numpy(ts + steps_offset)


def euler_trailing_timesteps(n: int) -> torch.Tensor:
    ts = np.round(np.arange(NUM_TRAIN_TIMESTEPS, 0, -NUM_TRAIN_TIMESTEPS / n)) - 1
    return torch.from_numpy(ts.astype(np.float32))


@dataclass
class Schedule:
    """State the reference keeps on `self` / `self.scheduler` after __init__."""
    total_alphas: torch.Tensor
    sigmas: torch.Tensor
    log_sigmas: torch.Tensor
    timesteps: torch.Tensor
    skip: int
    alphas_cumprod: torch.Tensor       # shifted: cat([1.0], abar) — index t == original t-1
    final_alpha_cumprod: torch.Tensor

    @staticmethod
    def make(num_sampling: int, kind: str = "ddim") -> "Schedule":
        abar = alphas_cumprod_table()
        sig = (1 - abar).sqrt() / abar.sqrt()
        ts = ddim_leading_timesteps(num_sampling) if kind == "ddim" else euler_trailing_timesteps(num_sampling)
        return Schedule(abar.clone(), sig, sig.log(), ts, NUM_TRAIN_TIMESTEPS // num_sampling,
                        torch.cat([torch.tensor([1.0]), abar]), abar[0].clone())

    def alpha(self, t) -> torch.Tensor:
        """StableDiffusion.alpha, latent_diffusion.py:88-90."""
        t = int(t)
        return self.alphas_cumprod[t] if t >= 0 else self.final_alpha_cumprod


def _state(t: float, in_scale: float, lam: float, c=(0, 0, 0, 0), d=(0, 0, 0, 0), second_order=0) -> StepStateC:
    s = StepStateC()
    s.t, s.in_scale = float(t), float(in_scale)
    s.coef.lambda_ = float(np.float32(schedule_lambda(lam)))  # a per-image table (cfgpp_set_guidance) overrides it
    s.coef.c0, s.coef.c1, s.coef.c2, s.coef.c3 = (float(x) for x in c)
    s.coef.d0, s.coef.d1, s.coef.d2, s.coef.d3 = (float(x) for x in d)
    s.coef.second_order = int(second_order)
    return s


def ddim_cfgpp_steps(sch: Schedule, cfg_guidance: float, sdxl_indexing: bool,
                     tables_on_device: bool = False) -> List[StepStateC]:
    """Sampling loop scalars. sdxl_indexing: `alphas_cumprod[t - skip]` with Python negative-index wrap on the last
    step (latent_sdxl.py:732-734); otherwise StableDiffusion.alpha() (negative -> final_alpha_cumprod).
    tables_on_device (Lightning, latent_sdxl.py:418): the table is a CUDA tensor there, and PyTorch casts a 0-dim
    CUDA operand of an fp16 tensor op to fp16 first — so the two scalars that multiply the fp16 eps tensors are
    rounded through fp16 (a CPU 0-dim operand, the SDXL / SD1.5 case, enters as an fp32 scalar instead)."""
    out = []
    for t in sch.timesteps.int():
        if sdxl_indexing:
            at, at_next = sch.alphas_cumprod[t], sch.alphas_cumprod[t - sch.skip]
        else:
            at, at_next = sch.alpha(t), sch.alpha(t - sch.skip)
        c0, c3 = (1 - at).sqrt(), (1 - at_next).sqrt()
        if tables_on_device:
            c0, c3 = c0.half().float(), c3.half().float()
        out.append(_state(float(t), 1.0, cfg_guidance, c=(c0, at.sqrt(), at_next.sqrt(), c3)))
    return out


def ddim_inversion_cfgpp_steps(sch: Schedule, cfg_guidance: float) -> List[StepStateC]:
    """InversionDDIMCFGpp.inversion scalars, latent_diffusion.py:897-908 (ascending t)."""
    out = []
    for t in reversed(sch.timesteps):
        at, at_prev = sch.alpha(t), sch.alpha(t - sch.skip)
        out.append(_state(float(t), 1.0, cfg_guidance,
                          c=((1 - at_prev).sqrt(), at_prev.sqrt(), at.sqrt(), (1 - at).sqrt())))
    return out


def sigma_to_t(sch: Schedule, sigma: torch.Tensor, quantize: bool = True) -> torch.Tensor:
    """SDXL.sigma_to_t (latent_sdxl.py:333-346, "taken from k_diffusion/external.py"): nearest index in the un-shifted
    sigma table (quantize=True, what the CFG++ solvers use) or the linearly interpolated fractional index."""
    total_sigmas = (1 - sch.total_alphas).sqrt() / sch.total_alphas.sqrt()
    dists = sigma - total_sigmas[:, None]
    if quantize:
        return dists.abs().argmin(dim=0).view(sigma.shape)
    low_idx = dists.ge(0).cumsum(dim=0).argmax(dim=0).clamp(max=total_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = total_sigmas[low_idx], total_sigmas[high_idx]
    w = ((low - sigma) / (low - high)).clamp(0, 1)
    t = (1 - w) * low_idx + w * high_idx
    return t.view(sigma.shape)


def expert_split(timesteps: torch.Tensor, denoising_end: float, nsteps: int) -> int:
    """Index k of the first step the second expert (the SDXL refiner) runs: the base runs steps [0, k), the refiner
    [k, nsteps). k = #{t in timesteps : t >= round(1000 * (1 - denoising_end))}, diffusers' rule for both the base
    pipeline's `denoising_end` and the refiner pipeline's `denoising_start`. Both experts must run at least one step."""
    if not 0.0 < denoising_end < 1.0:
        raise ValueError(f"denoising_end must lie strictly between 0 and 1, got {denoising_end}")
    cutoff = int(round(NUM_TRAIN_TIMESTEPS * (1.0 - denoising_end)))
    k = int((timesteps >= cutoff).sum())
    if not 1 <= k <= nsteps - 1:
        raise ValueError(f"denoising_end={denoising_end} leaves {k} of {nsteps} steps to the base model; each expert "
                         f"needs at least one step")
    return k


def dpmpp_2m_cfgpp_steps(sch: Schedule, cfg_guidance: float, restart_at: Optional[int] = None):
    """DPMpp2mCFGppSolver.reverse_process scalars (latent_sdxl.py:877-918). Returns (steps, sigma0).
    restart_at=k: entry k takes the first-order update, as the first step of a new call does — the hand-off to the
    SDXL refiner, which starts with no multistep history. Every other entry is unchanged."""
    alphas = sch.alphas_cumprod[sch.timesteps.int()]
    sigmas = (1 - alphas).sqrt() / alphas.sqrt()
    t_fn = lambda s: s.log().neg()  # noqa: E731
    out = []
    n = len(sch.timesteps) - 1
    for i in range(n):
        at, sigma = alphas[i], sigmas[i]
        c_in, c_out = at.clone().sqrt(), -sigma.clone()
        new_t = sigma_to_t(sch, sigma)
        t, t_next = t_fn(sigmas[i]), t_fn(sigmas[i + 1])
        h = t_next - t
        inv_sigma = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(sigmas[i].item(), dtype=torch.float32)
        if i == 0 or i == restart_at or sigmas[i + 1] == 0:
            out.append(_state(float(new_t), c_in, cfg_guidance, c=(c_out, inv_sigma, sigmas[i + 1], 0.0)))
        else:
            h_last = t - t_fn(sigmas[i - 1])
            r = h_last / h
            inv_2r = torch.tensor(1.0, dtype=torch.float32) / (2 * r)
            out.append(_state(float(new_t), c_in, cfg_guidance, c=(c_out, inv_sigma, sigmas[i + 1], 0.0),
                              d=(-torch.exp(-h), (-h).expm1(), inv_2r, torch.exp(-h)), second_order=1))
    return out, sigmas[0]


KD_SECOND_ORDER, KD_EXTRAP_GUIDED, KD_DIFF_GUIDED = 1, 2, 4   # cfgpp_step_coef.second_order bits
KD_NOISE, KD_2S_MID, KD_2S_FINAL = 8, 16, 32


def kd_steps(sigmas: torch.Tensor, timestep_fn, cfg_guidance: float, cfgpp: bool, second_order: bool = False,
             diff_guided: bool = False) -> List[StepStateC]:
    """Per-step scalars of the VE-cast ("k-diffusion") loops for the fused STEP_DPMPP2M_CFGPP family:
    Euler (latent_diffusion.py:699-719 / :326-330, latent_sdxl.py:787-808) and the Karras-sigma DPM++(2M) of SD v1.5
    (:847-877 / :470-487). `sigmas` ends with 0; `timestep_fn(sigma)` is the solver's `timestep()`.
    The UNet sees x / (sigma^2 + 1)^0.5 (a CPU-scalar divisor = an fp32 reciprocal multiply on CUDA) at t = timestep(sigma);
    den / ud = x - sigma eps; d = (x - extrap) / sigma.item() (again a reciprocal multiply)."""
    t_fn = lambda sg: sg.log().neg()  # noqa: E731
    one = torch.tensor(1.0, dtype=torch.float32)
    base = 0 if cfgpp else KD_EXTRAP_GUIDED
    out = []
    for i in range(len(sigmas) - 1):
        sigma = sigmas[i]
        in_scale = one / (sigma ** 2 + 1) ** 0.5
        inv_sigma = one / torch.tensor(sigma.item(), dtype=torch.float32)
        t = float(timestep_fn(sigma))
        c = (-sigma.clone(), inv_sigma, sigmas[i + 1], 0.0)
        if not second_order or i == 0 or sigmas[i + 1] == 0:
            out.append(_state(t, in_scale, cfg_guidance, c=c, second_order=base))
        else:
            h = t_fn(sigmas[i + 1]) - t_fn(sigmas[i])
            r = (t_fn(sigmas[i]) - t_fn(sigmas[i - 1])) / h
            out.append(_state(t, in_scale, cfg_guidance, c=c, d=(-torch.exp(-h), (-h).expm1(), one / (2 * r), torch.exp(-h)),
                              second_order=base | KD_SECOND_ORDER | (KD_DIFF_GUIDED if diff_guided else 0)))
    return out


def _ancestral_step(sigma_from, sigma_to, eta: float = 1.):
    """(sigma_down, sigma_up) — latent_diffusion.py:30-37 (same arithmetic on the same 0-dim tensors)."""
    if not eta:
        return sigma_to, 0.
    var_ratio = sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2
    sigma_up = min(sigma_to, eta * var_ratio ** 0.5)
    return (sigma_to ** 2 - sigma_up ** 2) ** 0.5, sigma_up


def kd_ancestral_steps(sigmas: torch.Tensor, timestep_fn, cfg_guidance: float, cfgpp: bool, two_s: bool = False):
    """Schedule entries of the ancestral VE-cast loops for the fused step kernel. Returns (entries, noise_slots):
    `euler_a(_cfg++)` (latent_diffusion.py:344-379 / :744-762): one entry per step, x' = den + d * sigma_down
    + noise * sigma_up; `dpm++_2s_a(_cfg++)` (:408-437 / :782-825, two_s=True): two entries (midpoint call, final
    call) per step with sigma_down > 0, the Euler form otherwise. A step with sigma_{i+1} > 0 consumes one noise slot,
    in loop order — the caller draws `noise_slots` tensors with `torch.randn_like` up front, which is the very
    sequence the reference's loop would draw."""
    t_fn = lambda sg: sg.log().neg()    # noqa: E731
    sigma_fn = lambda t: t.neg().exp()  # noqa: E731
    one = torch.tensor(1.0, dtype=torch.float32)
    base = 0 if cfgpp else KD_EXTRAP_GUIDED
    out, slot = [], 0
    for i in range(len(sigmas) - 1):
        sigma = sigmas[i]
        in_scale = one / (sigma ** 2 + 1) ** 0.5
        inv_sigma = one / torch.tensor(sigma.item(), dtype=torch.float32)
        t = float(timestep_fn(sigma))
        sigma_down, sigma_up = _ancestral_step(sigmas[i], sigmas[i + 1])
        noisy = bool(sigmas[i + 1] > 0)
        nbits = KD_NOISE if noisy else 0
        if not two_s or sigma_down == 0:
            out.append(_state(t, in_scale, cfg_guidance, c=(-sigma.clone(), inv_sigma, sigma_down, slot),
                              d=(0, 0, 0, sigma_up if noisy else 0.0), second_order=base | nbits))
        else:
            tt, t_next = t_fn(sigmas[i]), t_fn(sigma_down)
            r = 1 / 2
            h = t_next - tt
            s = tt + r * h
            sigma_s = sigma_fn(s)
            out.append(_state(t, in_scale, cfg_guidance, c=(-sigma.clone(), inv_sigma, 0.0, 0.0),
                              d=(sigma_fn(s) / sigma_fn(tt), (-h * r).expm1(), 0, 0), second_order=base | KD_2S_MID))
            out.append(_state(float(timestep_fn(sigma_s)), one / (sigma_s ** 2 + 1) ** 0.5, cfg_guidance,
                              c=(-sigma_s.clone(), 0.0, 0.0, slot),
                              d=(torch.exp(-h), sigma_fn(t_next) / sigma_fn(tt), (-h).expm1(), sigma_up if noisy else 0.0),
                              second_order=base | KD_2S_FINAL | nbits))
        slot += 1 if noisy else 0
    return out, slot


def ve_v_coefs(sigma: torch.Tensor):
    """(a, b) = (sqrt(abar), sqrt(1 - abar)) of a VE-cast state x at noise level sigma, abar = 1 / (1 + sigma^2): a = c_in
    (the model-input scale of `kd_steps`, same fp32 CPU ops) and b = sigma * c_in. Then eps = a v + b (c_in x), which is
    k-diffusion's VDenoiser (c_skip = 1 / (sigma^2 + 1), c_out = -sigma c_in) rewritten as an eps prediction."""
    c_in = torch.tensor(1.0, dtype=torch.float32) / (sigma ** 2 + 1) ** 0.5
    return c_in, sigma * c_in


def v_pred_coefs(method: int, steps: List[StepStateC]) -> np.ndarray:
    """Per schedule entry (a, b) = (sqrt(abar), sqrt(1 - abar)) of the noise level the entry's own update assigns to the
    state the UNet sees, float32 [n, 2]. A v-prediction model's output becomes eps = fp16(fp32(a v) + fp32(b x_in))
    before the step (see v_to_eps).
      DDIM family (sampling, inversion, plain CFG): the update's Tweedie divisor c1 = sqrt(abar) and c0 = sqrt(1 - abar)
        (sampling: abar = alpha(t); inversion: abar = alpha(t - skip), the level the state sits at).
      VE-cast family: ve_v_coefs(sigma) of the entry's sigma = -c0, i.e. a = in_scale, b = sigma * in_scale — each of
        the two UNet calls of a DPM-Solver++(2S) step with its own sigma."""
    out = np.zeros((len(steps), 2), dtype=np.float32)
    for i, st in enumerate(steps):
        if method == STEP_DPMPP2M_CFGPP:
            a = np.float32(st.in_scale)
            out[i] = (a, np.float32(-st.coef.c0) * a)
        else:
            out[i] = (st.coef.c1, st.coef.c0)
    return out


def v_to_eps(v: torch.Tensor, x_in: torch.Tensor, a, b) -> torch.Tensor:
    """eps = fp16(fp32(a v) + fp32(b x_in)) — the fused step kernel's conversion (two fp32 products, an fp32 sum, no
    FMA) on fp16 tensors v and x_in (the UNet's fp16 input); a, b fp32 scalars."""
    return (v.float() * float(a) + x_in.float() * float(b)).half()


def to_c_array(steps: List[StepStateC]):
    arr = (StepStateC * len(steps))()
    for i, s in enumerate(steps):
        arr[i] = s
    return arr
