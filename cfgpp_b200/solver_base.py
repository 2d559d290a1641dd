"""What the SD (latent_diffusion.py) and SDXL (latent_sdxl.py) solver families share: the registry factory, the
schedule attributes the reference keeps on `self`, and the VAE front and back end."""
from __future__ import annotations

from typing import Any

import torch

from . import kdiffusion as K
from . import schedule as S
from .lora import LoraMixin


def registry():
    """(__SOLVER__, register_solver, get_solver) of one solver family (latent_diffusion.py:13-26)."""
    solvers = {}

    def register_solver(name: str):
        def wrapper(cls):
            if solvers.get(name, None) is not None:
                raise ValueError(f"Solver {name} already registered.")
            solvers[name] = cls
            return cls
        return wrapper

    def get_solver(name: str, **kwargs):
        if name not in solvers:
            raise ValueError(f"Solver {name} does not exist.")
        return solvers[name](**kwargs)

    return solvers, register_solver, get_solver


class _Scheduler:
    """The two attributes of the diffusers scheduler object the reference touches."""
    def __init__(self, sch: S.Schedule, device):
        self.timesteps = sch.timesteps.to(device)
        self.alphas_cumprod = sch.alphas_cumprod
        self.final_alpha_cumprod = sch.final_alpha_cumprod


CONTROL_KWARGS = ("controlnet", "control_image", "controlnet_conditioning_scale", "control_guidance_start",
                  "control_guidance_end")


def refuse_control(kwargs: dict, what: str) -> None:
    """The inversion / editing solvers take no ControlNet, no IP-Adapter and no T2I-Adapter."""
    if kwargs.get("controlnet") is not None or kwargs.get("control_image") is not None:
        raise ValueError(f"{what} does not take a ControlNet (text-to-image solvers only)")
    refuse_ip_adapter(kwargs, what)
    if kwargs.get("t2i_adapter") is not None or kwargs.get("t2i_adapter_image") is not None:
        raise ValueError(f"{what} does not take a T2I-Adapter (text-to-image solvers only)")


def refuse_ip_adapter(kwargs: dict, what: str) -> None:
    if kwargs.get("ip_adapter") is not None or kwargs.get("ip_adapter_image") is not None:
        raise ValueError(f"{what} does not take an IP-Adapter (SD v1.5 / SDXL text-to-image solvers only)")


class IPRequest:
    """The IP-Adapter of one sample() call: the adapter, the image embeds of its batch (one per prompt) and the
    scale."""

    def __init__(self, adapter, embeds: torch.Tensor, scale: float):
        self.adapter, self.embeds, self.scale = adapter, embeds, float(scale)


def ip_request(kwargs: dict, batch: int):
    """The IPRequest that sample()'s `ip_adapter=`, `ip_adapter_image=` (one image, broadcast, or one per prompt) and
    `ip_adapter_scale=` ask for, or None."""
    ad, image = kwargs.get("ip_adapter"), kwargs.get("ip_adapter_image")
    if ad is None and image is None:
        return None
    if ad is None or image is None:
        raise ValueError("ip_adapter and ip_adapter_image go together")
    return IPRequest(ad, ad.image_embeds(image, batch), kwargs.get("ip_adapter_scale", 1.0))


class SolverBase(K.KDiffusionMixin, LoraMixin):
    """The host class provides `vae`, `dtype` and `sample`."""
    _control = None  # the ControlRequest of the running sample() call (controlnet.control_request), else None

    def _controlled(self, kwargs: dict, batch: int, lat_h: int, lat_w: int, run):
        """run() under the ControlNet, IP-Adapter and T2I-Adapter that sample()'s keyword arguments ask for (none: the
        engine is detached)."""
        from .controlnet import control_request
        from .t2i_adapter import t2i_request
        ip = ip_request(kwargs, batch)
        if ip is not None and ip.adapter.base_cfg != self.unet.cfg:
            raise ValueError(f"ip_adapter was built for {ip.adapter.base_cfg.name}, this solver runs "
                             f"{self.unet.cfg.name} (IP-Adapter: SD v1.5 and SDXL)")
        self._control = control_request(kwargs, batch, 8 * lat_h, 8 * lat_w, self.device)
        t2i = None
        if kwargs.get("t2i_adapter") is not None or kwargs.get("t2i_adapter_image") is not None:
            t2i = t2i_request(kwargs, self.unet.cfg, batch, 8 * lat_h, 8 * lat_w)
        if ip is not None:  # the engine's set-up (bind_control) attaches it; without one it detaches any adapter
            self.unet.ip_request = ip
        if t2i is not None:  # likewise; the word starts on for the un-fused steps (a schedule sets its own)
            self.unet.t2i_request = t2i
            self.unet.set_t2i_active(True)
        try:
            return run()
        finally:
            self._control = None
            if ip is not None:
                self.unet.ip_request = None
            if t2i is not None:
                self.unet.t2i_request = None

    def _control_entries(self, steps):
        """The conditioning scale of every entry of `steps`, or None when uncontrolled."""
        return None if self._control is None else self._control.entry_scales(steps)

    def _control_step(self, i: int, n: int) -> None:
        """Sampler step i of n runs un-fused next: its UNet calls take that step's conditioning scale and T2I word."""
        if self._control is not None:
            self.unet.set_control_scale(self._control.step_scale(i, n))
        t2i = getattr(self.unet, "t2i_request", None)
        if t2i is not None:
            self.unet.set_t2i_active(t2i.step_on(i, n))

    def _init_schedule(self, num_sampling: int, kind: str, device):
        """Sampling parameters (latent_diffusion.py:69-80, latent_sdxl.py:56-67 / :407-418)."""
        self._sch = S.Schedule.make(num_sampling, kind)
        self.total_alphas = self._sch.total_alphas
        self.sigmas = self._sch.sigmas
        self.log_sigmas = self._sch.log_sigmas
        self.skip = self._sch.skip
        self.final_alpha_cumprod = self._sch.final_alpha_cumprod
        self.scheduler = _Scheduler(self._sch, device)

    def __call__(self, *args: Any, **kwargs: Any) -> Any:
        self.sample(*args, **kwargs)

    @torch.no_grad()
    def encode(self, x):
        return self.vae.encode(x, self.dtype)

    def decode(self, zt):
        return self.vae.decode(zt).float()

    @torch.no_grad()
    def to_image(self, zt):
        """The decoded latent as images in [0, 1] on the host, (B, 3, H, W)."""
        return (self.decode(zt) / 2 + 0.5).clamp(0, 1).detach().cpu()
