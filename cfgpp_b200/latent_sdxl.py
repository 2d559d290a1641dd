"""SDXL / SDXL-Lightning CFG++ solvers on the Blackwell-native backend.

Mirror of the reference's `latent_sdxl.py` solver API for the hot path named by BASELINE.json — same registry
(`register_solver` / `get_solver`, latent_sdxl.py:15-28), same class / method names and argument meaning
(`SDXL.sample` :200-266, `reverse_process` :715-755 / :843-858 / :864-930, `predict_noise` :167-185,
`initialize_latent` :268-299, `sigma_to_t` :333-346), same errors (ValueError for unknown / duplicate solver,
AssertionError for Lightning with cfg_guidance != 1, NotImplementedError for unknown init methods) — but the UNet
forward, the CFG++ guidance mix and the scheduler update run in hand-written sm_90a CUDA behind the C ABI
(include/cfgpp_b200.h). With `callback_fn=None` a whole trajectory is enqueued as NFE replays of one CUDA graph with
no host synchronisation (`NativeUNet.run_trajectory`); with a callback the un-fused seam (`NativeUNet.callback_step`:
`predict_noise` + `apply_step`) is used so that `z0t` / `zt` are materialised and may be replaced by the callback,
exactly like the reference loop.

Registered here: ddim_cfg++, ddim_cfg++_lightning, dpm++_2m_cfgpp (the solvers of SURVEY.md §8a) and, from §8 f1,
dpm++_2m_cfgpp_lightning (:932-952), ddim_edit_cfg++ (:954-1025, both loops on the fused step modes), euler_cfg++ and
euler_cfg++_lightning (:757-836: fused VE-cast trajectories, kdiffusion.py; the op-by-op torch form only with a callback).
A plain-CFG solver and its CFG++ twin share one body: the DDIM ones differ in the class attributes `step_mode` /
`inversion_mode`, the Euler ones in their sigma table and `cfgpp`. A Lightning solver lists SDXLLightning first in its
bases, for its checkpoint, its schedule and its guidance check.
The VAE (decode and encode, vae.py, SURVEY §8 f2) and the two CLIP text towers (text_encoder.py, §8 f3) run on the
native backend too; `text_encoders=` / `vae=` accept replacements.
"""
from __future__ import annotations

import warnings
from typing import Optional, Tuple

import torch

from . import kdiffusion as K
from . import schedule as S
from .batching import (draw_latents, encode_prompts, guidance_table, guidance_values, normalize_batch,
                       sdxl_added_conditions)
from .conditioning import SyntheticTextEncoder
from .text_encoder import CLIPTextConfig, ClipConditioner, get_conditioner
from .config import UNetConfig, sdxl_config, sdxl_refiner_config
from .engine import NativeUNet
from .lora import LoraMixin, is_lora_file, read_lora
from .solver_base import SolverBase, refuse_control, refuse_ip_adapter, registry
from .weights import load_safetensors_state_dict, synthetic_state_dict

__SOLVER__, register_solver, get_solver = registry()

_ENGINES = {}


def resolve_state_dict(model_key: str, cfg: UNetConfig, device):
    """`*.safetensors` path -> real weights; 'synthetic[:seed]' -> seeded synthetic; anything else (an HF hub id:
    nothing can be downloaded here) -> synthetic with a warning."""
    if model_key.endswith(".safetensors"):
        return load_safetensors_state_dict(model_key, device=device)
    seed = 1234
    if model_key.startswith("synthetic"):
        if ":" in model_key:
            seed = int(model_key.split(":", 1)[1])
    else:
        warnings.warn(f"no checkpoint for '{model_key}' is available offline; using seeded synthetic UNet weights "
                      f"(pass a diffusers-format *.safetensors path as model_key for real weights)")
    return synthetic_state_dict(cfg, seed=seed, device=device)


def get_engine(model_key: str, cfg: UNetConfig, device, state_dict=None, lora: Optional[str] = None) -> NativeUNet:
    """The engine of (model_key, config, device), built once and shared. `lora`: a LoRA file that belongs to the
    model's identity (SDXL-Lightning distributed as a LoRA): such an engine is cached apart from the plain base model's
    and carries the adapter at scale 1."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("cfgpp_b200 solvers run on CUDA (sm_90a) only — there is no CPU fallback on the product "
                           "path; the CPU eager baseline lives in oracle/ and bench.py")
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    key = (model_key if lora is None else f"{model_key}+lora:{lora}", cfg.name, idx)
    ent = _ENGINES.get(key)
    # an explicit state_dict is part of the identity: the entry keeps a strong reference to it and compares with `is`
    # (an id() of a dead dict can be recycled by a different one)
    if ent is not None and ent[1] is state_dict:
        return ent[0]
    # same key, other weights: the cache entry is replaced; the old engine (5 GB) is destroyed by NativeUNet.__del__
    # as soon as the last solver holding it goes away
    sd = state_dict if state_dict is not None else resolve_state_dict(model_key, cfg, torch.device("cuda", idx))
    eng = NativeUNet(cfg, sd, torch.device("cuda", idx))
    if lora is not None:
        eng.add_lora(read_lora(lora, cfg), 1.0)
    _ENGINES[key] = (eng, state_dict)
    return eng


def release_engines():
    """Destroy every cached engine (packed weights + workspace) — the cache otherwise lives as long as the process."""
    for eng, _ in _ENGINES.values():
        eng.close()
    _ENGINES.clear()


def default_text_encoders(cfg: UNetConfig, device):
    """(text_enc_1, text_enc_2) for a UNet config: CLIP-L + OpenCLIP bigG for the real SDXL widths (768 + 1280 = 2048,
    pooled 1280), proportionally narrow towers for the test-sized configs; widths that are not multiples of the 64-wide
    CLIP head fall back to the shape-only stand-in of conditioning.py."""
    d2 = cfg.pooled_dim
    d1 = cfg.cross_attention_dim - d2
    if d1 <= 0:
        d1 = cfg.cross_attention_dim // 2
        d2 = cfg.cross_attention_dim - d1
    if (d1, d2, cfg.pooled_dim) == (768, 1280, 1280):
        return (get_conditioner("clip_l", device, "sdxl"), get_conditioner("clip_bigg", device, "sdxl"))
    if d1 % 64 or d2 % 64 or cfg.pooled_dim % 8:
        return (SyntheticTextEncoder(d1, 0), SyntheticTextEncoder(d2, cfg.pooled_dim))

    def small(name, d, proj, act, pad):
        return CLIPTextConfig(name=name, vocab_size=1024, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=2,
                              num_attention_heads=d // 64, hidden_act=act, projection_dim=proj, pad_token_id=pad)
    return (get_conditioner("", device, "sdxl", cfg=small(f"clip_{d1}", d1, 0, "quick_gelu", 1023)),
            get_conditioner("", device, "sdxl", cfg=small(f"clip_{d2}_proj", d2, cfg.pooled_dim, "gelu", 0)))


def _prepare_engine(eng: NativeUNet, zt, uc, c, added_cond_kwargs, force: bool = False, control=None):
    """Prepare `eng` for zt's shape and bind the prompt, with `control`'s ControlNet attached (None: detached)."""
    if eng.cfg.addition_embed_type == "text_time":
        eng.bind_control(control, zt, uc, c, added_cond_kwargs['text_embeds'], added_cond_kwargs['time_ids'],
                         force=force)
    else:
        eng.bind_control(control, zt, uc, c, force=force)


REFINER_SOLVERS = ("ddim", "ddim_cfg++", "dpm++_2m_cfgpp")


class SDXLRefiner(LoraMixin):
    """The second expert of SDXL 1.0 (stabilityai/stable-diffusion-xl-refiner-1.0): a UNet that takes over a base
    trajectory for its last, low-noise steps ("ensemble of experts"; diffusers' `denoising_end` on the base pipeline,
    `denoising_start` on the refiner's). Pass it to `sample(refiner=...)` of one of REFINER_SOLVERS.

    It holds only its UNet engine (cached next to the base's in the engine cache, keyed by the config name) and,
    optionally, its text tower: None uses the base solver's second tower (OpenCLIP bigG), the refiner's only one, so no
    second copy is loaded. The base solver's VAE decodes the refined latent."""

    def __init__(self, model_key: str = "stabilityai/stable-diffusion-xl-refiner-1.0", device='cuda',
                 unet_config: Optional[UNetConfig] = None, state_dict=None, text_encoder=None):
        self.cfg = unet_config or sdxl_refiner_config()
        self.unet = get_engine(model_key, self.cfg, device, state_dict)
        self.text_enc = text_encoder


class SDXL(SolverBase):
    schedule_kind = "ddim"
    quantize = True
    supports_refiner = False  # the fused DDIM / DPM++ trajectories of REFINER_SOLVERS hand over to a refiner
    step_mode = S.STEP_DDIM_CFG       # fused step mode of the DDIM sampling loop
    inversion_mode = S.STEP_DDIM_CFG  # ... and of the inversion loop

    def __init__(self,
                 solver_config,
                 model_key: str = "stabilityai/stable-diffusion-xl-base-1.0",
                 dtype=torch.float16,
                 device='cuda',
                 unet_config: Optional[UNetConfig] = None,
                 state_dict=None,
                 text_encoders=None,
                 vae=None,
                 lora: Optional[str] = None):
        self.device = device
        self.dtype = dtype
        self.cfg = unet_config or sdxl_config()
        self.unet = get_engine(model_key, self.cfg, device, state_dict, lora)

        # CLIP text towers on the native backend (text_encoder.py; the reference takes pipe.text_encoder /
        # pipe.text_encoder_2, latent_sdxl.py:46-49). Pass `text_encoders=(fn1, fn2)`, prompt -> (hidden, pooled), to override.
        self.text_enc_1, self.text_enc_2 = text_encoders or default_text_encoders(self.cfg, device)
        if vae is None:
            # AutoencoderKL decoder on the native backend (vae.py; the reference loads madebyollin/sdxl-vae-fp16-fix,
            # latent_sdxl.py:44). Pass `vae=` (any object with decode(zt) / encode(x, dtype)) to override.
            from .vae import get_vae
            vae = get_vae("sdxl_vae", device)
        self.vae = vae
        self.vae_scale_factor = self.cfg.vae_scale_factor
        self.default_sample_size = self.cfg.sample_size
        self._init_schedule(solver_config.num_sampling, self.schedule_kind, device)

    def alpha(self, t):
        return self.scheduler.alphas_cumprod[t] if t >= 0 else self.final_alpha_cumprod

    @torch.no_grad()
    def _text_embed(self, prompt, text_enc, clip_skip, batch: int = 1):
        """One prompt (broadcast to `batch` rows) or a list of prompts, one row each."""
        if isinstance(text_enc, ClipConditioner):
            return encode_prompts(lambda p: text_enc(p, self.device, clip_skip=clip_skip), prompt, batch, True)
        return encode_prompts(lambda p: text_enc(p, self.device), prompt, batch)

    @torch.no_grad()
    def get_text_embed(self, null_prompt_1, prompt_1, null_prompt_2=None, prompt_2=None, clip_skip=None,
                       batch: int = 1):
        prompt_embed_1, pool_prompt_embed = self._text_embed(prompt_1, self.text_enc_1, clip_skip, batch)
        if prompt_2 is None:
            prompt_embed = [prompt_embed_1]
        else:
            prompt_embed_2, pool_prompt_embed = self._text_embed(prompt_2, self.text_enc_2, clip_skip, batch)
            prompt_embed = [prompt_embed_1, prompt_embed_2]
        null_embed_1, pool_null_embed = self._text_embed(null_prompt_1, self.text_enc_1, clip_skip, batch)
        if null_prompt_2 is None:
            null_embed = [null_embed_1]
        else:
            null_embed_2, pool_null_embed = self._text_embed(null_prompt_2, self.text_enc_2, clip_skip, batch)
            null_embed = [null_embed_1, null_embed_2]
        null_prompt_embeds = torch.concat(null_embed, dim=-1)
        prompt_embeds = torch.concat(prompt_embed, dim=-1)
        return null_prompt_embeds, prompt_embeds, pool_null_embed, pool_prompt_embed

    # ---- the seam: batched (uncond + cond) UNet forward on the native backend -----------------------------------
    def _prepare(self, zt, uc, c, added_cond_kwargs, force: bool = False):
        _prepare_engine(self.unet, zt, uc, c, added_cond_kwargs, force, self._control)

    def predict_noise(self, zt, t, uc, c, added_cond_kwargs, in_scale: float = 1.0):
        if uc is None or c is None:
            # single-branch paths of the reference (latent_sdxl.py:169-176) are never taken by the CFG++ solvers
            uc = c if uc is None else uc
            c = uc if c is None else c
        self._prepare(zt, uc, c, added_cond_kwargs)
        return self.unet.predict_noise(zt, float(t), in_scale)

    def _get_add_time_ids(self, original_size, crops_coords_top_left, target_size, dtype, text_encoder_projection_dim,
                          aesthetic_score: Optional[float] = None, cfg: Optional[UNetConfig] = None):
        """`cfg` (default: this solver's UNet) decides the form, as diffusers' `requires_aesthetics_score` does: a UNet
        of 5 time ids (the SDXL refiner) takes (original size, crop top-left, aesthetic score) in place of the
        base's (original size, crop top-left, target size)."""
        cfg = cfg or self.cfg
        if cfg.num_time_ids == 5:
            add_time_ids = list(original_size + crops_coords_top_left + (aesthetic_score,))
        else:
            add_time_ids = list(original_size + crops_coords_top_left + target_size)
        passed_add_embed_dim = cfg.addition_time_embed_dim * len(add_time_ids) + text_encoder_projection_dim
        expected_add_embed_dim = cfg.projection_class_embeddings_input_dim
        assert expected_add_embed_dim == passed_add_embed_dim, (
            f"Model expects an added time embedding vector of length {expected_add_embed_dim}, but a vector of "
            f"{passed_add_embed_dim} was created. The model has an incorrect config.")
        return torch.tensor([add_time_ids], dtype=dtype)

    def _time_id_pair(self, dtype, pool, original_size, crops_coords_top_left, target_size, negative_original_size,
                      negative_crops_coords_top_left, negative_target_size):
        """(negative, positive) time ids of a sample() call; the negative ones are the positive ones unless both
        negative sizes are given."""
        kw = dict(dtype=dtype, text_encoder_projection_dim=int(pool.shape[-1]))
        add_time_ids = self._get_add_time_ids(original_size, crops_coords_top_left, target_size, **kw)
        if negative_original_size is None or negative_target_size is None:
            return add_time_ids, add_time_ids
        return self._get_add_time_ids(negative_original_size, negative_crops_coords_top_left, negative_target_size,
                                      **kw), add_time_ids

    def sample(self,
               prompt1=["", ""],
               prompt2=["", ""],
               cfg_guidance: float = 5.0,
               original_size: Optional[Tuple[int, int]] = None,
               crops_coords_top_left: Tuple[int, int] = (0, 0),
               target_size: Optional[Tuple[int, int]] = None,
               negative_original_size: Optional[Tuple[int, int]] = None,
               negative_crops_coords_top_left: Tuple[int, int] = (0, 0),
               negative_target_size: Optional[Tuple[int, int]] = None,
               clip_skip: Optional[int] = None,
               refiner: Optional[SDXLRefiner] = None,
               denoising_end: float = 0.8,
               aesthetic_score: float = 6.0,
               negative_aesthetic_score: float = 2.5,
               **kwargs):
        """Batched: `prompt1[1]` / `prompt2[1]` one string or B strings, the null prompts one string (broadcast) or B
        strings, `cfg_guidance` a float or B floats (one per image, applied in the fused step kernel), `zT` None or
        (B,4,h,w); without zT the B latents are drawn one image at a time, so image i does not depend on B. Mismatched
        lengths raise ValueError. Returns (B, 3, H, W).

        `refiner`: an SDXLRefiner that runs the steps after `denoising_end` (a fraction of the schedule, see
        schedule.expert_split) in the same trajectory; the image is decoded once, after it. The refiner is conditioned
        as diffusers' refiner pipeline conditions it: `prompt1` through its text tower, time ids (original size, crop
        top-left, `aesthetic_score`) and, for the uncond row, `negative_aesthetic_score`.

        ControlNet: `controlnet=` (a controlnet.ControlNet), `control_image=` (B or 1, 3, H, W) in [0, 1] at the output
        size, `controlnet_conditioning_scale=`, `control_guidance_start=` / `control_guidance_end=` (diffusers' meaning,
        over the whole schedule); a refiner runs uncontrolled.

        IP-Adapter: `ip_adapter=` (an ip_adapter.IPAdapter for this UNet), `ip_adapter_image=` (one image, broadcast,
        or one per prompt), `ip_adapter_scale=` (1.0); not with `refiner=`."""
        if refiner is not None:
            self._check_refiner()
            refuse_ip_adapter(kwargs, "sample(refiner=...)")
        size = self.default_sample_size * self.vae_scale_factor
        original_size, target_size = original_size or (size, size), target_size or (size, size)

        B, p, cfg_guidance = normalize_batch({"prompt1[0]": prompt1[0], "prompt1[1]": prompt1[1],
                                              "prompt2[0]": prompt2[0], "prompt2[1]": prompt2[1]},
                                             cfg_guidance, kwargs.get('zT'))
        (null_prompt_embeds, prompt_embeds, pool_null_embed, pool_prompt_embed) = self.get_text_embed(
            p["prompt1[0]"], p["prompt1[1]"], p["prompt2[0]"], p["prompt2[1]"], clip_skip, batch=B)
        negative_add_time_ids, add_time_ids = self._time_id_pair(
            prompt_embeds.dtype, pool_prompt_embed, original_size, crops_coords_top_left, target_size,
            negative_original_size, negative_crops_coords_top_left, negative_target_size)

        # per image: the uncond row takes the negative pooled embedding / time ids unless its lambda is 0 or 1
        add_text_embeds, add_time_ids = sdxl_added_conditions(pool_null_embed, pool_prompt_embed, negative_add_time_ids,
                                                              add_time_ids, cfg_guidance, B)

        add_cond_kwargs = {'text_embeds': add_text_embeds.to(self.device), 'time_ids': add_time_ids.to(self.device)}

        if refiner is not None:
            kwargs.update(refiner=refiner, denoising_end=denoising_end, refiner_cond=self.refiner_conditions(
                refiner, p["prompt1[0]"], p["prompt1[1]"], cfg_guidance, original_size, crops_coords_top_left,
                negative_original_size or original_size, negative_crops_coords_top_left, aesthetic_score,
                negative_aesthetic_score, clip_skip, B))
        zT = kwargs.get('zT')
        lat = (zT.shape[2], zT.shape[3]) if zT is not None else (target_size[1] // self.vae_scale_factor,
                                                                 target_size[0] // self.vae_scale_factor)
        return self.to_image(self._controlled(kwargs, B, *lat, lambda: self.reverse_process(
            null_prompt_embeds, prompt_embeds, cfg_guidance, add_cond_kwargs, target_size, **kwargs)))

    @torch.no_grad()
    def refiner_conditions(self, refiner: SDXLRefiner, null_prompt, prompt, cfg_guidance, original_size,
                           crops_coords_top_left, negative_original_size, negative_crops_coords_top_left,
                           aesthetic_score, negative_aesthetic_score, clip_skip=None, batch: int = 1):
        """(uc, c, added_cond_kwargs) of the refiner, following diffusers' StableDiffusionXLImg2ImgPipeline (stated
        here: diffusers is not a dependency): its encode_prompt zips [prompt, prompt_2] with its single tokenizer, so
        only the `prompt1` pair reaches the one text tower (bigG), whose penultimate hidden state is the context and
        whose text_embeds are the pooled embedding; the time ids take the aesthetic form; the rows are assembled per
        image by the same lambda rule as the base's."""
        enc = refiner.text_enc or self.text_enc_2
        uc, pool_null = self._text_embed(null_prompt, enc, clip_skip, batch)
        c, pool = self._text_embed(prompt, enc, clip_skip, batch)
        proj = int(pool.shape[-1])
        time_ids = self._get_add_time_ids(original_size, crops_coords_top_left, None, c.dtype, proj,
                                          aesthetic_score, refiner.cfg)
        negative_time_ids = self._get_add_time_ids(negative_original_size, negative_crops_coords_top_left, None,
                                                   c.dtype, proj, negative_aesthetic_score, refiner.cfg)
        text_embeds, time_ids = sdxl_added_conditions(pool_null, pool, negative_time_ids, time_ids, cfg_guidance,
                                                      batch)
        return uc, c, {'text_embeds': text_embeds.to(self.device), 'time_ids': time_ids.to(self.device)}

    def _check_refiner(self):
        if not self.supports_refiner or self.schedule_kind == "lightning":
            raise ValueError(f"an SDXL refiner runs with the solvers {', '.join(REFINER_SOLVERS)} only, not with "
                             f"{type(self).__name__}")

    def _hand_off(self, kwargs, nsteps: int):
        """(refiner, its (uc, c, added_cond_kwargs), k) of a reverse_process call given `refiner=`, else None."""
        refiner = kwargs.get('refiner')
        if refiner is None:
            return None
        self._check_refiner()
        k = S.expert_split(self._sch.timesteps, kwargs.get('denoising_end', 0.8), nsteps)
        return refiner, kwargs['refiner_cond'], k

    def initialize_latent(self, method: str = 'random', src_img: Optional[torch.Tensor] = None,
                          add_cond_kwargs: Optional[dict] = None, **kwargs):
        if method == 'random':
            size = kwargs.get('size', (1, 4, 128, 128))
            z = draw_latents(size).to(self.device)  # CPU generator, then H2D — latent_sdxl.py:288-289
        elif method == 'random_kdiffusion':
            size = kwargs.get('latent_dim', (1, 4, 128, 128))
            sigmas = kwargs.get('sigmas', [14.6146])
            z = draw_latents(size).to(self.device)
            z = z * (sigmas[0] ** 2 + 1) ** 0.5
        elif method == 'ddim':
            assert src_img is not None, "src_img must be provided for inversion"
            z = self.inversion(self.encode(src_img.to(self.dtype).to(self.device)), kwargs.get('uc'), kwargs.get('c'),
                               kwargs.get('cfg_guidance', 0.0), add_cond_kwargs)
        elif method == 'npi':
            assert src_img is not None, "src_img must be provided for inversion"
            z = self.inversion(self.encode(src_img.to(self.dtype).to(self.device)), kwargs.get('c'), kwargs.get('c'),
                               1.0, add_cond_kwargs)
        else:
            raise NotImplementedError
        return z

    def reverse_process(self, *args, **kwargs):
        raise NotImplementedError

    @torch.no_grad()
    def inversion(self, z0, uc, c, cfg_guidance, add_cond_kwargs):
        """DDIM inversion (latent_sdxl.py:301-324) on the fused `inversion_mode` with the fp16 VAE latent as state:
        plain CFG takes Tweedie and renoise both with the guided eps, CFG++ (:955-1025) Tweedie with eps_uc."""
        if cfg_guidance == 0.0 or cfg_guidance == 1.0:
            add_cond_kwargs['text_embeds'] = add_cond_kwargs['text_embeds'][-1].unsqueeze(0)
            add_cond_kwargs['time_ids'] = add_cond_kwargs['time_ids'][-1].unsqueeze(0)
        steps = S.ddim_inversion_cfgpp_steps(self._sch, cfg_guidance)
        z0 = z0.clone().to(self.device)
        _, zt = self._run_trajectory(self.inversion_mode, z0.dtype, steps, z0, (uc, c, add_cond_kwargs))
        return zt

    def sigma_to_t(self, sigma, quantize=None):
        quantize = self.quantize if quantize is None else quantize
        return S.sigma_to_t(self._sch, sigma, quantize)

    # ---- trajectory: fused, or step by step under a callback; optionally handed to a refiner ----------------------
    def _run_trajectory(self, method, state_dtype, steps, z_init, cond, callback_fn=None, cfg_guidance=None,
                        hand_off=None):
        """(z0t, zt) after the last step from `z_init` under `cond` = (uc, c, added_cond_kwargs): the DDIM family returns
        the Tweedie estimate z0t, DPM++ the state zt. `cfg_guidance`: a per-image sequence goes to the step kernel's
        guidance table.
        `hand_off` (see _hand_off): steps [k, n) of the same table run on the refiner's engine, which continues from
        the base's state in the sampler's own parameterization; both engines are set up before the first step, so
        the hand-off is a device-to-device copy with no host synchronisation. The step index a callback sees runs
        0..n-1 across both."""
        table, scales = guidance_table(cfg_guidance), self._control_entries(steps)
        if hand_off is None and callback_fn is None:
            _prepare_engine(self.unet, z_init, *cond, force=True, control=self._control)  # re-binds its prompt
            return self.unet.run_trajectory(method, state_dtype, steps, z_init, table, control_scales=scales)
        experts = [(self.unet, cond, self._control, scales)]
        k = len(steps)
        if hand_off is not None:
            refiner, refiner_cond, k = hand_off
            experts.append((refiner.unet, refiner_cond, None, None))  # the refiner runs uncontrolled
        for e, e_cond, e_control, e_scales in experts:
            _prepare_engine(e, z_init, *e_cond, force=True, control=e_control)
            e.set_schedule(method, state_dtype, steps, table, e_scales)
        eng = self.unet
        eng.set_state(z_init)
        if callback_fn is None:
            eng.run_steps(0, k)
            eng, base = experts[1][0], eng
            eng.set_state(base.get_state(0))
            eng.run_steps(k, len(steps) - k)
            return eng.get_state(1), eng.get_state(0)
        for i, st in enumerate(steps):
            if i == k:
                eng, base = experts[1][0], eng
                eng.set_state(base.get_state(0))
            if scales is not None and i < k:
                eng.set_control_scale(scales[i])
            z0t, zt = eng.callback_step(i, st)
            kw = {'z0t': z0t.detach(), 'zt': zt.detach(), 'decode': self.decode}
            kw = callback_fn(i, torch.tensor(int(st.t), device=self.device), kw)
            eng.set_state(kw['zt'])
            z0t = kw['z0t']
        return z0t, eng.get_state(0)


class SDXLLightning(SDXL):
    """SDXL-Lightning: the distilled UNet (or its LoRA on the base UNet) on the trailing schedule, guidance off. A
    Lightning solver lists this class first in its bases, so that this __init__ and the guidance check run in place of
    the plain sampler's."""
    schedule_kind = "lightning"

    def __init__(self,
                 solver_config,
                 base_model_key: str = "stabilityai/stable-diffusion-xl-base-1.0",
                 light_model_ckpt: str = "ckpt/sdxl_lightning_4step_unet.safetensors",
                 dtype=torch.float16,
                 device='cuda',
                 **kwargs):
        import os
        if os.path.exists(light_model_ckpt) and is_lora_file(light_model_ckpt):
            # the LoRA distribution (sdxl_lightning_*step_lora.safetensors): the base UNet with the file as an adapter
            SDXL.__init__(self, solver_config, model_key=base_model_key, dtype=dtype, device=device,
                          lora=light_model_ckpt, **kwargs)
            return
        key = light_model_ckpt if os.path.exists(light_model_ckpt) else "synthetic:4321"
        if key.startswith("synthetic"):
            warnings.warn(f"Lightning checkpoint '{light_model_ckpt}' not found; using seeded synthetic UNet weights")
        SDXL.__init__(self, solver_config, model_key=key, dtype=dtype, device=device, **kwargs)

    def reverse_process(self, null_prompt_embeds, prompt_embeds, cfg_guidance, add_cond_kwargs, shape=(1024, 1024),
                        callback_fn=None, **kwargs):
        assert all(g == 1.0 for g in guidance_values(cfg_guidance)), "CFG should be turned off in the lightning version"
        return super().reverse_process(null_prompt_embeds, prompt_embeds, cfg_guidance, add_cond_kwargs, shape,
                                       callback_fn, **kwargs)


###########################################
# Samplers: plain CFG (the baselines the paper compares against, SURVEY §8 f4) and CFG++
###########################################


@register_solver('ddim')
class BaseDDIM(SDXL):
    """latent_sdxl.py:425-467: fp32 state, fused trajectory, renoise with the guided eps."""
    supports_refiner = True

    def reverse_process(self, null_prompt_embeds, prompt_embeds, cfg_guidance, add_cond_kwargs, shape=(1024, 1024),
                        callback_fn=None, **kwargs):
        """`refiner=`, `refiner_cond=` (uc, c, added_cond_kwargs), `denoising_end=`: hand the trajectory to an SDXL
        refiner (sample() builds the conditioning)."""
        b = null_prompt_embeds.shape[0]
        zt = kwargs.get('zT')
        if zt is None:
            zt = self.initialize_latent(size=(b, 4, shape[1] // self.vae_scale_factor, shape[0] // self.vae_scale_factor))
        steps = S.ddim_cfgpp_steps(self._sch, cfg_guidance, sdxl_indexing=True,
                                   tables_on_device=(self.schedule_kind == "lightning"))
        # fp32 state: zt comes from torch.randn (fp32) and promotes every update (latent_sdxl.py:289, 741-744)
        z0t, _ = self._run_trajectory(self.step_mode, torch.float32, steps, zt.float(),
                                      (null_prompt_embeds, prompt_embeds, add_cond_kwargs), callback_fn, cfg_guidance,
                                      self._hand_off(kwargs, len(steps)))
        return z0t


@register_solver("ddim_cfg++")
class BaseDDIMCFGpp(BaseDDIM):
    step_mode = S.STEP_DDIM_CFGPP


@register_solver('ddim_lightning')
class BaseDDIMLight(SDXLLightning, BaseDDIM):
    pass


@register_solver('ddim_cfg++_lightning')
class BaseDDIMCFGppLight(SDXLLightning, BaseDDIMCFGpp):
    pass


@register_solver('euler')
class Euler(SDXL):
    """Karras Euler (VE casted), plain CFG, Karras sigmas (latent_sdxl.py:469-517)."""
    cfgpp = False

    def euler_sigmas(self):
        ts = self.total_sigmas()
        return K.get_sigmas_karras(len(self.scheduler.timesteps), ts.min(), ts.max(), rho=7.)

    @torch.no_grad()
    def reverse_process(self, null_prompt_embeds, prompt_embeds, cfg_guidance, add_cond_kwargs, shape=(1024, 1024),
                        callback_fn=None, **kwargs):
        sigmas = self.euler_sigmas()
        zt = kwargs.get('xT')
        if zt is None and kwargs.get('zT') is not None:  # an N(0,1) draw, as every other solver accepts it
            zt = kwargs['zT'].to(self.device) * (sigmas[0] ** 2 + 1) ** 0.5
        if zt is None:
            zt_dim = (null_prompt_embeds.shape[0], 4, shape[1] // self.vae_scale_factor,
                      shape[0] // self.vae_scale_factor)
            zt = self.initialize_latent(method="random_kdiffusion", latent_dim=zt_dim, sigmas=sigmas)
        z0t, _ = K.euler_cfgpp_loop(self, zt.to(torch.float16), sigmas, cfg_guidance,
                                    (null_prompt_embeds, prompt_embeds, add_cond_kwargs), callback_fn, cfgpp=self.cfgpp)
        return z0t


@register_solver('euler_cfg++')
class EulerCFGpp(Euler):
    """Karras Euler (VE casted) with CFG++ on the sampling timesteps' own sigmas (latent_sdxl.py:757-808): the native
    UNet behind `predict_noise`, the Euler update in torch (kdiffusion.py)."""
    cfgpp = True

    def euler_sigmas(self):
        sigmas = self.total_sigmas()[torch.round(self.scheduler.timesteps.cpu()).int()]
        return torch.cat([sigmas, torch.tensor([0.0])])


@register_solver('euler_lightning')
class EulerLight(SDXLLightning, Euler):
    pass


@register_solver('euler_cfg++_lightning')
class EulerCFGppLight(SDXLLightning, EulerCFGpp):
    pass


@register_solver('dpm++_2m_cfgpp')
class DPMpp2mCFGppSolver(SDXL):
    supports_refiner = True

    def reverse_process(self, null_prompt_embeds, prompt_embeds, cfg_guidance, add_cond_kwargs, shape=(1024, 1024),
                        callback_fn=None, **kwargs):
        b = null_prompt_embeds.shape[0]
        # a refiner starts with no multistep history: its first step takes the first-order update
        hand_off = self._hand_off(kwargs, len(self._sch.timesteps) - 1)
        steps, sigma0 = S.dpmpp_2m_cfgpp_steps(self._sch, cfg_guidance,
                                               restart_at=None if hand_off is None else hand_off[2])
        x = kwargs.get('zT')
        if x is None:
            x = self.initialize_latent(method='random', size=(b, 4, shape[1] // self.vae_scale_factor,
                                                              shape[0] // self.vae_scale_factor))
        x = x.to(torch.float16)
        x = x * sigma0  # fp16 tensor x 0-dim fp32 -> fp16 (latent_sdxl.py:882-884)
        _, x = self._run_trajectory(S.STEP_DPMPP2M_CFGPP, torch.float16, steps, x,
                                    (null_prompt_embeds, prompt_embeds, add_cond_kwargs), callback_fn, cfg_guidance,
                                    hand_off)
        return x


@register_solver('dpm++_2m_cfgpp_lightning')
class DPMpp2mCFGppLightningSolver(SDXLLightning, DPMpp2mCFGppSolver):
    pass


@register_solver("ddim_edit")
class EditWardSwapDDIM(SDXL):
    """Three-prompt front end of the editing solvers (prompt = [null, source, target]) — latent_sdxl.py:570-655 — and
    the plain-CFG edit loop (:656-707): plain inversion under the source prompt, plain DDIM under the target prompt,
    both through `alpha()` with the fp16 VAE latent as state (fused step mode STEP_DDIM_CFG)."""

    def reverse_process(self, null_prompt_embeds, src_prompt_embeds, tgt_prompt_embed, cfg_guidance,
                        add_src_cond_kwargs, add_tgt_cond_kwargs, callback_fn=None, **kwargs):
        zt = self.initialize_latent(method='ddim', src_img=kwargs.get('src_img', None), uc=null_prompt_embeds,
                                    c=src_prompt_embeds, cfg_guidance=cfg_guidance,
                                    add_cond_kwargs=add_src_cond_kwargs)
        steps = S.ddim_cfgpp_steps(self._sch, cfg_guidance, sdxl_indexing=False)
        z0t, _ = self._run_trajectory(self.step_mode, zt.dtype, steps, zt,
                                      (null_prompt_embeds, tgt_prompt_embed, add_tgt_cond_kwargs), callback_fn)
        return z0t

    def sample(self,
               prompt1=["", "", ""],
               prompt2=["", "", ""],
               cfg_guidance: float = 5.0,
               original_size: Optional[Tuple[int, int]] = None,
               crops_coords_top_left: Tuple[int, int] = (0, 0),
               target_size: Optional[Tuple[int, int]] = None,
               negative_original_size: Optional[Tuple[int, int]] = None,
               negative_crops_coords_top_left: Tuple[int, int] = (0, 0),
               negative_target_size: Optional[Tuple[int, int]] = None,
               clip_skip: Optional[int] = None,
               **kwargs):
        refuse_control(kwargs, "ddim_edit")
        if kwargs.get('refiner') is not None:
            self._check_refiner()
        size = self.default_sample_size * self.vae_scale_factor
        original_size, target_size = original_size or (size, size), target_size or (size, size)

        (null_prompt_embeds, src_prompt_embeds, pool_null_embed, pool_src) = self.get_text_embed(
            prompt1[0], prompt1[1], prompt2[0], prompt2[1], clip_skip)
        (_, tgt_prompt_embeds, _, pool_tgt) = self.get_text_embed(prompt1[0], prompt1[2], prompt2[0], prompt2[2],
                                                                  clip_skip)
        negative_add_time_ids, add_time_ids = self._time_id_pair(
            src_prompt_embeds.dtype, pool_src, original_size, crops_coords_top_left, target_size,
            negative_original_size, negative_crops_coords_top_left, negative_target_size)
        # one image: the reference's lambda in {0, 1} rule on the scalar guidance (latent_sdxl.py:249-257)
        add_src, add_tgt = pool_src, pool_tgt
        if cfg_guidance != 0.0 and cfg_guidance != 1.0:
            add_src = torch.cat([pool_null_embed, add_src], dim=0)
            add_tgt = torch.cat([pool_null_embed, add_tgt], dim=0)
            add_time_ids = torch.cat([negative_add_time_ids, add_time_ids], dim=0)
        add_src_cond_kwargs = {'text_embeds': add_src.to(self.device), 'time_ids': add_time_ids.to(self.device)}
        add_tgt_cond_kwargs = {'text_embeds': add_tgt.to(self.device), 'time_ids': add_time_ids.to(self.device)}

        return self.to_image(self.reverse_process(null_prompt_embeds, src_prompt_embeds, tgt_prompt_embeds,
                                                  cfg_guidance, add_src_cond_kwargs, add_tgt_cond_kwargs, **kwargs))


@register_solver("ddim_edit_cfg++")
class EditWardSwapDDIMCFGpp(EditWardSwapDDIM):
    """CFG++ inversion under the source prompt (Tweedie with eps_uc, renoise with the guided eps), then CFG++ DDIM
    sampling under the target prompt — latent_sdxl.py:955-1025. Both loops index the schedule through `alpha()`
    (negative t -> final_alpha_cumprod) and carry the fp16 VAE latent, so they run as the two fused step modes the
    SD v1.5 `ddim_inversion_cfg++` uses."""
    step_mode, inversion_mode = S.STEP_DDIM_CFGPP, S.STEP_DDIM_INV_CFGPP


if __name__ == "__main__":
    print(f"Possble solvers: {[x for x in __SOLVER__.keys()]}")
