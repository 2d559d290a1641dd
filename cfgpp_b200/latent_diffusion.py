"""Stable Diffusion v1.5 and 2.x CFG++ solvers on the Blackwell-native backend.

Mirror of the reference's `latent_diffusion.py` solver API for the hot path: registry (:13-26), `StableDiffusion`
base (:54-241: `alpha`, `get_text_embed`, `predict_noise`, `inversion`, `initialize_latent`; `encode` / `decode` and
the registry factory are shared with the SDXL family in solver_base.py),
`ddim_cfg++` (:621-679) and `ddim_inversion_cfg++` (:882-957). Same names, argument meaning and errors; the UNet
forward, CFG++ mix and DDIM update run in hand-written sm_90a CUDA behind include/cfgpp_b200.h.
SURVEY §8 f1 (the rest of the CFG++ `--method` surface): `ddim_edit_cfg++` (:959-1010) on the same fused step modes;
`euler_cfg++` (:682-724), `euler_a_cfg++` (:727-768), `dpm++_2s_a_cfg++` (:771-827), `dpm++_2m_cfg++` (:830-879) as
fused VE-cast trajectories (kdiffusion.py: the ancestral ones with their noise drawn up front); the op-by-op torch
form over `predict_noise` runs when a callback is installed. A plain-CFG DDIM solver and its CFG++ twin share one body
and differ in the class attributes `step_mode` / `inversion_mode` (the fused step kernel's modes).

SD 2.x (`unet_config=sd2_config()` / `sd2_base_config()`) runs on the same solvers: the UNet differs only in its
config, and a v-prediction model's output is turned into eps inside the fused step (see schedule.v_pred_coefs).

dtype note (reference promotion rules, SURVEY Appendix C.5): `ddim_cfg++` keeps an fp32 latent state (zT is a fp32
`torch.randn`); `ddim_inversion_cfg++` starts from the fp16 VAE latent, so both its inversion loop and the following
sampling loop run with an fp16 state — every update op rounds to fp16, which the fused step kernel reproduces.
"""
from __future__ import annotations

from typing import Any, Optional

import torch

from . import kdiffusion as K
from . import schedule as S
from .batching import draw_latents, encode_prompts, guidance_table, normalize_batch
from .conditioning import SyntheticTextEncoder
from .text_encoder import CLIPTextConfig, get_conditioner
from .config import UNetConfig, sd15_config
from .latent_sdxl import get_engine
from .solver_base import SolverBase, refuse_control, registry

__SOLVER__, register_solver, get_solver = registry()


def default_text_encoder(cfg: UNetConfig, device):
    """CLIP-L (hidden 768) for SD v1.5, OpenCLIP ViT-H (hidden 1024) for SD 2.x; a proportionally narrow tower for the
    test-sized configs."""
    d = cfg.cross_attention_dim
    if d == 768:
        return get_conditioner("clip_l", device, "sd15")
    if d == 1024:
        return get_conditioner("clip_h", device, "sd15")
    if d % 64:
        return SyntheticTextEncoder(d, 0)
    small = CLIPTextConfig(name=f"clip_{d}", vocab_size=1024, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=2,
                           num_attention_heads=d // 64, pad_token_id=1023)
    return get_conditioner("", device, "sd15", cfg=small)


class StableDiffusion(SolverBase):
    step_mode = S.STEP_DDIM_CFG       # fused step mode of the sampling loop
    inversion_mode = S.STEP_DDIM_CFG  # ... and of the inversion loop

    def __init__(self,
                 solver_config,
                 model_key: str = "runwayml/stable-diffusion-v1-5",
                 device: Optional[torch.device] = None,
                 **kwargs):
        self.device = device
        self.dtype = kwargs.get("pipe_dtype", torch.float16)
        self.cfg: UNetConfig = kwargs.get("unet_config") or sd15_config()
        # SD 2.0-v / 2.1: the UNet predicts v. The fused steps convert it to eps in the step kernel; predict_noise and
        # the VE-cast seam (_k_denoise) convert the same way, so every seam still hands eps to the sampler arithmetic.
        self.v_prediction = self.cfg.prediction_type == "v_prediction"
        self.unet = get_engine(model_key, self.cfg, device, kwargs.get("state_dict"))
        # CLIP-L text tower on the native backend (text_encoder.py; the reference takes pipe.text_encoder,
        # latent_diffusion.py:65-66). Pass `text_encoder=fn`, prompt -> (hidden (1,77,D), None), to override.
        self.text_encoder = kwargs.get("text_encoder") or default_text_encoder(self.cfg, device)
        self.vae = kwargs.get("vae")
        if self.vae is None:
            # AutoencoderKL decoder on the native backend (vae.py; the reference uses pipe.vae, latent_diffusion.py:64)
            from .vae import get_vae
            self.vae = get_vae("sd15_vae", device)
        self._init_schedule(solver_config.num_sampling, "ddim", device)

    def sample(self, *args: Any, **kwargs: Any) -> Any:
        raise NotImplementedError("Solver must implement sample() method.")

    def alpha(self, t):
        return self._sch.alpha(t)

    @torch.no_grad()
    def get_text_embed(self, null_prompt, prompt, batch: int = 1):
        """One prompt each (a string is broadcast to `batch` rows) or lists of prompts, one row per prompt."""
        from .text_encoder import ClipConditioner
        takes_list = isinstance(self.text_encoder, ClipConditioner)
        enc = lambda p: self.text_encoder(p, self.device)  # noqa: E731
        null_text_embed, _ = encode_prompts(enc, null_prompt, batch, takes_list)
        text_embed, _ = encode_prompts(enc, prompt, batch, takes_list)
        return null_text_embed, text_embed

    def batch_inputs(self, prompt, cfg_guidance, zT=None):
        """(uc, c, cfg_guidance, zT) of a batched text-to-image call: `prompt[1]` one string or B strings, `prompt[0]`
        one string (broadcast) or B strings, `cfg_guidance` a float or B floats (one per image, applied in the fused
        step kernel), `zT` None or (B,4,h,w). Mismatched lengths raise ValueError."""
        B, p, cfg_guidance = normalize_batch({"prompt[0]": prompt[0], "prompt[1]": prompt[1]}, cfg_guidance, zT)
        uc, c = self.get_text_embed(null_prompt=p["prompt[0]"], prompt=p["prompt[1]"], batch=B)
        return uc, c, cfg_guidance, zT

    def _prepare(self, zt, uc, c, force: bool = False):
        self.unet.bind_control(self._control, zt, uc, c, force=force)

    def model_output(self, zt: torch.Tensor, t: torch.Tensor, uc: torch.Tensor, c: torch.Tensor):
        """The UNet's raw (uncond, cond) output at input zt: eps, or v for a v-prediction model."""
        if uc is None or c is None:
            uc = c if uc is None else uc
            c = uc if c is None else c
        self._prepare(zt, uc, c)
        return self.unet.predict_noise(zt, float(t))

    def predict_noise(self, zt: torch.Tensor, t: torch.Tensor, uc: torch.Tensor, c: torch.Tensor):
        out_uc, out_c = self.model_output(zt, t, uc, c)
        if not self.v_prediction:
            return out_uc, out_c
        at = self.alpha(t)
        a, b = at.sqrt(), (1 - at).sqrt()
        x_in = zt.to(out_uc.device, torch.float16)
        return S.v_to_eps(out_uc, x_in, a, b), S.v_to_eps(out_c, x_in, a, b)

    def _run(self, method, steps, z_init, uc, c, callback_fn=None, cfg_guidance=None):
        """(z0t, zt) of a DDIM-family trajectory. `cfg_guidance`: a per-image sequence goes to the step kernel's
        guidance table; a float (or None) leaves the steps' scalar in charge."""
        self._prepare(z_init, uc, c, force=True)  # every trajectory re-binds its prompt
        eng, table, scales = self.unet, guidance_table(cfg_guidance), self._control_entries(steps)
        if callback_fn is None:
            return eng.run_trajectory(method, z_init.dtype, steps, z_init, table, control_scales=scales)
        eng.set_schedule(method, z_init.dtype, steps, table)
        eng.set_state(z_init)
        for i, st in enumerate(steps):
            if scales is not None:
                eng.set_control_scale(scales[i])
            z0t, zt = eng.callback_step(i, st)
            kw = {'z0t': z0t.detach(), 'zt': zt.detach(), 'decode': self.decode}
            kw = callback_fn(i, torch.tensor(int(st.t), device=self.device), kw)
            z0t = kw['z0t']
            eng.set_state(kw['zt'])
        return z0t, eng.get_state(0)

    @torch.no_grad()
    def inversion(self, z0: torch.Tensor, uc: torch.Tensor, c: torch.Tensor, cfg_guidance: float = 1.0):
        """DDIM inversion (latent_diffusion.py:160-182) on the fused `inversion_mode`: plain CFG takes Tweedie and
        renoise both with the guided eps; CFG++ (:897-908) takes Tweedie with eps_uc. Same scalars for both."""
        steps = S.ddim_inversion_cfgpp_steps(self._sch, cfg_guidance)
        _, zt = self._run(self.inversion_mode, steps, z0.clone().to(self.device), uc, c)
        return zt

    def initialize_latent(self, method: str = 'random', src_img: Optional[torch.Tensor] = None, **kwargs):
        if method == 'ddim':
            z = self.inversion(self.encode(src_img.to(self.dtype).to(self.device)), kwargs.get('uc'), kwargs.get('c'),
                               cfg_guidance=kwargs.get('cfg_guidance', 0.0))
        elif method == 'npi':
            z = self.inversion(self.encode(src_img.to(self.dtype).to(self.device)), kwargs.get('c'), kwargs.get('c'),
                               cfg_guidance=1.0)
        elif method == 'random':
            size = kwargs.get('latent_dim', (1, 4, self.cfg.sample_size, self.cfg.sample_size))
            z = draw_latents(size).to(self.device)  # CPU generator, then H2D — latent_diffusion.py:199-200
        elif method == 'random_kdiffusion':
            size = kwargs.get('latent_dim', (1, 4, self.cfg.sample_size, self.cfg.sample_size))
            sigmas = kwargs.get('sigmas', [14.6146])
            z = draw_latents(size).to(self.device)
            z = z * (sigmas[0] ** 2 + 1) ** 0.5
        else:
            raise NotImplementedError
        return z


###########################################
# DDIM: plain CFG (the baselines the paper compares against, SURVEY §8 f4) and CFG++
###########################################

@register_solver("ddim")
class BaseDDIM(StableDiffusion):
    """Basic DDIM solver for SD with plain CFG (latent_diffusion.py:247-299), fused trajectory."""

    def reverse_process(self, uc, c, cfg_guidance, zt, callback_fn=None):
        steps = S.ddim_cfgpp_steps(self._sch, cfg_guidance, sdxl_indexing=False)
        z0t, _ = self._run(self.step_mode, steps, zt, uc, c, callback_fn, cfg_guidance)
        return z0t

    def sample(self, cfg_guidance=7.5, prompt=["", ""], callback_fn=None, **kwargs):
        """Batched: see StableDiffusion.batch_inputs. Returns (B, 3, H, W). ControlNet: `controlnet=` (a
        controlnet.ControlNet), `control_image=` (B or 1, 3, H, W) in [0, 1] at the output size,
        `controlnet_conditioning_scale=`, `control_guidance_start=` / `control_guidance_end=` (diffusers' meaning).
        IP-Adapter: `ip_adapter=` (an ip_adapter.IPAdapter for this UNet), `ip_adapter_image=` (one image, broadcast,
        or one per prompt), `ip_adapter_scale=` (1.0)."""
        uc, c, cfg_guidance, zt = self.batch_inputs(prompt, cfg_guidance, kwargs.get('zT'))
        if zt is None:
            zt = self.initialize_latent(latent_dim=(uc.shape[0], 4, self.cfg.sample_size, self.cfg.sample_size))
        return self.to_image(self._controlled(kwargs, uc.shape[0], zt.shape[2], zt.shape[3],
                                              lambda: self.reverse_process(uc, c, cfg_guidance, zt, callback_fn)))


@register_solver("ddim_inversion")
class InversionDDIM(BaseDDIM):
    """Reconstruction / editing after plain-CFG inversion (latent_diffusion.py:506-558)."""

    def sample(self, src_img, cfg_guidance=7.5, prompt=["", ""], callback_fn=None, **kwargs):
        refuse_control(kwargs, "ddim_inversion")
        uc, c = self.get_text_embed(null_prompt=prompt[0], prompt=prompt[1])
        zt = self.initialize_latent(method='ddim', src_img=src_img, uc=uc, c=c, cfg_guidance=cfg_guidance)
        return self.to_image(self.reverse_process(uc, c, cfg_guidance, zt, callback_fn))


@register_solver("ddim_edit")
class EditWordSwapDDIM(InversionDDIM):
    """Editing via WordSwap after plain-CFG inversion (latent_diffusion.py:561-612)."""

    def sample(self, src_img, cfg_guidance=7.5, prompt=["", "", ""], callback_fn=None, **kwargs):
        refuse_control(kwargs, "ddim_edit")
        uc, src_c = self.get_text_embed(null_prompt=prompt[0], prompt=prompt[1])
        _, tgt_c = self.get_text_embed(null_prompt=prompt[0], prompt=prompt[2])
        zt = self.initialize_latent(method='ddim', src_img=src_img, uc=uc, c=src_c, cfg_guidance=cfg_guidance)
        return self.to_image(self.reverse_process(uc, tgt_c, cfg_guidance, zt, callback_fn))


@register_solver("ddim_cfg++")
class BaseDDIMCFGpp(BaseDDIM):
    """DDIM solver for SD with CFG++ (text-to-image)."""
    step_mode = S.STEP_DDIM_CFGPP


@register_solver("ddim_inversion_cfg++")
class InversionDDIMCFGpp(InversionDDIM):
    """Reconstruction after CFG++ inversion (Tweedie with eps_uc, renoise with the guided eps) and CFG++ sampling."""
    step_mode, inversion_mode = S.STEP_DDIM_CFGPP, S.STEP_DDIM_INV_CFGPP


@register_solver("ddim_edit_cfg++")
class EditWordSwapDDIMCFGpp(EditWordSwapDDIM):
    """Editing via WordSwap after inversion: CFG++ inversion under the source prompt, CFG++ sampling under the target
    prompt (latent_diffusion.py:959-1010). Both loops run as fused trajectories with an fp16 state."""
    step_mode, inversion_mode = S.STEP_DDIM_CFGPP, S.STEP_DDIM_INV_CFGPP


class _KarrasCFGpp(StableDiffusion):
    """Shared front / back end of the VE-cast samplers: Karras sigmas over the NFE steps, x ~ N(0, sigma_0^2 + 1) in
    fp16, decode of either the last Tweedie estimate or the final state (latent_diffusion.py:688-697, 720-724)."""
    adopt_callback = True
    decode_state = False  # True: decode x (dpm++ variants), False: decode the last denoised (euler variants)

    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        raise NotImplementedError

    def karras_sigmas(self):
        ts = self.total_sigmas()
        return K.get_sigmas_karras(len(self.scheduler.timesteps), ts.min(), ts.max(), rho=7.)

    @torch.no_grad()
    def reverse_process(self, uc, c, cfg_guidance, x=None, callback_fn=None, noise=None):
        """`x`: a ready (scaled) start state; `noise`: an N(0,1) draw to scale (the `zT` every solver accepts)."""
        sigmas = self.karras_sigmas()
        if x is None and noise is not None:
            x = noise.to(self.device) * (sigmas[0] ** 2 + 1) ** 0.5
        if x is None:
            x = self.initialize_latent(method="random_kdiffusion", sigmas=sigmas,
                                       latent_dim=(uc.shape[0], 4, self.cfg.sample_size, self.cfg.sample_size))
        return self._loop(x.to(torch.float16), sigmas, cfg_guidance, (uc, c), callback_fn)

    def sample(self, cfg_guidance, prompt=["", ""], callback_fn=None, **kwargs):
        """Batched: see StableDiffusion.batch_inputs. Ancestral methods draw each step's noise with `randn_like` over
        the whole batch, as the reference's loop would on a batched x: their images are not the serial runs' images."""
        uc, c, cfg_guidance, zt = self.batch_inputs(prompt, cfg_guidance, kwargs.get('zT'))
        ref = kwargs.get('xT') if kwargs.get('xT') is not None else zt
        h, w = (ref.shape[2], ref.shape[3]) if ref is not None else (self.cfg.sample_size,) * 2
        denoised, x = self._controlled(kwargs, uc.shape[0], h, w, lambda: self.reverse_process(
            uc, c, cfg_guidance, kwargs.get('xT'), callback_fn, zt))
        return self.to_image(x if self.decode_state else denoised)


@register_solver("euler_cfg++")
class EulerCFGppSolver(_KarrasCFGpp):
    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        # the reference binds the callback's return values to unused names here (:713-719): nothing is adopted
        return K.euler_cfgpp_loop(self, x, sigmas, cfg_guidance, cond, callback_fn, adopt_callback=False)


@register_solver("euler_a_cfg++")
class EulerAncestralCFGppSolver(_KarrasCFGpp):
    """Karras Euler (VE casted) + ancestral sampling."""
    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        return K.euler_cfgpp_loop(self, x, sigmas, cfg_guidance, cond, callback_fn, ancestral=True,
                                  adopt_callback=False)


@register_solver("dpm++_2s_a_cfg++")
class DPMpp2sAncestralCFGppSolver(_KarrasCFGpp):
    decode_state = True

    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        return K.dpmpp_2s_a_cfgpp_loop(self, x, sigmas, cfg_guidance, cond, callback_fn)


@register_solver("dpm++_2m_cfg++")
class DPMpp2mCFGppSolver(_KarrasCFGpp):
    decode_state = True

    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        return K.dpmpp_2m_cfgpp_karras_loop(self, x, sigmas, cfg_guidance, cond, callback_fn)


@register_solver("euler")
class EulerCFGSolver(_KarrasCFGpp):
    """Karras Euler (VE casted), plain CFG (latent_diffusion.py:302-346)."""
    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        return K.euler_cfgpp_loop(self, x, sigmas, cfg_guidance, cond, callback_fn, adopt_callback=False, cfgpp=False)


@register_solver("euler_a")
class EulerAncestralCFGSolver(_KarrasCFGpp):
    """Karras Euler + ancestral sampling, plain CFG (latent_diffusion.py:349-390)."""
    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        return K.euler_cfgpp_loop(self, x, sigmas, cfg_guidance, cond, callback_fn, ancestral=True,
                                  adopt_callback=False, cfgpp=False)


@register_solver("dpm++_2s_a")
class DPMpp2sAncestralCFGSolver(_KarrasCFGpp):
    """DPM-Solver++(2S) ancestral, plain CFG (latent_diffusion.py:393-451)."""
    decode_state = True

    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        return K.dpmpp_2s_a_cfgpp_loop(self, x, sigmas, cfg_guidance, cond, callback_fn, cfgpp=False)


@register_solver("dpm++_2m")
class DPMpp2mCFGSolver(_KarrasCFGpp):
    """DPM-Solver++(2M), plain CFG (latent_diffusion.py:454-503)."""
    decode_state = True

    def _loop(self, x, sigmas, cfg_guidance, cond, callback_fn):
        return K.dpmpp_2m_cfgpp_karras_loop(self, x, sigmas, cfg_guidance, cond, callback_fn, cfgpp=False)


if __name__ == "__main__":
    print(f"Possble solvers: {[x for x in __SOLVER__.keys()]}")
