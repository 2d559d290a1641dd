"""AutoencoderKL decoder on the Blackwell-native backend (SURVEY.md §8 f2).

Replaces `self.vae.decode(zt / self.vae.config.scaling_factor).sample` of the reference (latent_sdxl.py:155-164 with
`madebyollin/sdxl-vae-fp16-fix`, :44; latent_diffusion.py:123-129 with the SD v1.5 VAE, :64): post_quant_conv, the
decoder's resnets / mid-block attention / upsamplers and conv_out run through the C ABI (`cfgpp_vae_*`) on the same
wgmma conv / GEMM and GroupNorm kernels as the UNet. Weights use the diffusers AutoencoderKL key names
(`post_quant_conv.*`, `decoder.*`); no checkpoint exists offline, so the default weights are seeded synthetic ones
(a `*.safetensors` VAE file is loaded when given). The ENCODER half — `vae.encode(x).latent_dist.sample() *
scaling_factor`, the front end of the inversion / editing solvers (latent_sdxl.py:151-152, latent_diffusion.py:117-121)
— runs on the same handle (`cfgpp_vae_encode`: stride-2 TMA convs for the downsamplers, the posterior's noise drawn by
the caller from the CUDA generator like diffusers' `randn_tensor`). There is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import math
import warnings
from ctypes import byref, c_double, c_float, c_int, c_size_t
from dataclasses import dataclass
from typing import Dict, List, Tuple

import torch

from . import _native as nv
from .conditioning import LatentPreviewDecoder
from .config import CFGPP_MAX_LEVELS


@dataclass(frozen=True)
class VAEConfig:
    name: str = "sdxl_vae"
    latent_channels: int = 4
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    norm_num_groups: int = 32
    scaling_factor: float = 0.13025  # SDXL (latent_sdxl.py:163 reads vae.config.scaling_factor)


def sdxl_vae_config() -> VAEConfig:
    return VAEConfig()


def sd15_vae_config() -> VAEConfig:
    return VAEConfig(name="sd15_vae", scaling_factor=0.18215)  # the literal of latent_diffusion.py:127


def tiny_vae_config() -> VAEConfig:
    """Same topology (4 levels = x8 upsampling) at test-sized widths."""
    return VAEConfig(name="tiny_vae", block_out_channels=(64, 64, 128, 128), layers_per_block=1)


VAE_CONFIGS = {"sdxl_vae": sdxl_vae_config, "sd15_vae": sd15_vae_config, "tiny_vae": tiny_vae_config}


class VaeDescC(ctypes.Structure):
    _fields_ = [("latent_channels", c_int), ("out_channels", c_int), ("num_levels", c_int),
                ("block_out_channels", c_int * CFGPP_MAX_LEVELS), ("layers_per_block", c_int),
                ("norm_num_groups", c_int), ("scaling_factor", c_float)]


def to_vae_desc(cfg: VAEConfig) -> VaeDescC:
    d = VaeDescC()
    d.latent_channels, d.out_channels, d.num_levels = cfg.latent_channels, cfg.out_channels, len(cfg.block_out_channels)
    for i, c in enumerate(cfg.block_out_channels):
        d.block_out_channels[i] = c
    d.layers_per_block, d.norm_num_groups, d.scaling_factor = cfg.layers_per_block, cfg.norm_num_groups, cfg.scaling_factor
    return d


Spec = Tuple[str, Tuple[int, ...], str]


def _vae_resnet(prefix: str, cin: int, cout: int) -> List[Spec]:
    out = [(f"{prefix}.norm1.weight", (cin,), "norm_w"), (f"{prefix}.norm1.bias", (cin,), "norm_b"),
           (f"{prefix}.conv1.weight", (cout, cin, 3, 3), "w"), (f"{prefix}.conv1.bias", (cout,), "b"),
           (f"{prefix}.norm2.weight", (cout,), "norm_w"), (f"{prefix}.norm2.bias", (cout,), "norm_b"),
           (f"{prefix}.conv2.weight", (cout, cout, 3, 3), "w_res"), (f"{prefix}.conv2.bias", (cout,), "b")]
    if cin != cout:
        out += [(f"{prefix}.conv_shortcut.weight", (cout, cin, 1, 1), "w"), (f"{prefix}.conv_shortcut.bias", (cout,), "b")]
    return out


def vae_decoder_param_specs(cfg: VAEConfig) -> List[Spec]:
    """(diffusers key, shape, init kind) of post_quant_conv + decoder, in module order."""
    boc = cfg.block_out_channels
    ct = boc[-1]
    out: List[Spec] = [("post_quant_conv.weight", (4, 4, 1, 1), "w_pq"), ("post_quant_conv.bias", (4,), "b"),
                       ("decoder.conv_in.weight", (ct, cfg.latent_channels, 3, 3), "w"), ("decoder.conv_in.bias", (ct,), "b")]
    out += _vae_resnet("decoder.mid_block.resnets.0", ct, ct)
    a = "decoder.mid_block.attentions.0"
    out += [(f"{a}.group_norm.weight", (ct,), "norm_w"), (f"{a}.group_norm.bias", (ct,), "norm_b")]
    for n, kind in (("to_q", "w_qk"), ("to_k", "w_qk"), ("to_v", "w"), ("to_out.0", "w_res")):
        out += [(f"{a}.{n}.weight", (ct, ct), kind), (f"{a}.{n}.bias", (ct,), "b")]
    out += _vae_resnet("decoder.mid_block.resnets.1", ct, ct)
    rev = list(reversed(boc))
    cout = rev[0]
    for i, c in enumerate(rev):
        cin, cout = cout, c
        for j in range(cfg.layers_per_block + 1):
            out += _vae_resnet(f"decoder.up_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i != len(rev) - 1:
            out += [(f"decoder.up_blocks.{i}.upsamplers.0.conv.weight", (cout, cout, 3, 3), "w"),
                    (f"decoder.up_blocks.{i}.upsamplers.0.conv.bias", (cout,), "b")]
    out += [("decoder.conv_norm_out.weight", (boc[0],), "norm_w"), ("decoder.conv_norm_out.bias", (boc[0],), "norm_b"),
            ("decoder.conv_out.weight", (cfg.out_channels, boc[0], 3, 3), "w_out"), ("decoder.conv_out.bias", (cfg.out_channels,), "b")]
    return out


def vae_encoder_param_specs(cfg: VAEConfig) -> List[Spec]:
    """(diffusers key, shape, init kind) of encoder + quant_conv, in module order."""
    boc = cfg.block_out_channels
    ct = boc[-1]
    out: List[Spec] = [("encoder.conv_in.weight", (boc[0], cfg.out_channels, 3, 3), "w"), ("encoder.conv_in.bias", (boc[0],), "b")]
    cout = boc[0]
    for i, c in enumerate(boc):
        cin, cout = cout, c
        for j in range(cfg.layers_per_block):
            out += _vae_resnet(f"encoder.down_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i != len(boc) - 1:
            out += [(f"encoder.down_blocks.{i}.downsamplers.0.conv.weight", (cout, cout, 3, 3), "w"),
                    (f"encoder.down_blocks.{i}.downsamplers.0.conv.bias", (cout,), "b")]
    out += _vae_resnet("encoder.mid_block.resnets.0", ct, ct)
    a = "encoder.mid_block.attentions.0"
    out += [(f"{a}.group_norm.weight", (ct,), "norm_w"), (f"{a}.group_norm.bias", (ct,), "norm_b")]
    for n, kind in (("to_q", "w_qk"), ("to_k", "w_qk"), ("to_v", "w"), ("to_out.0", "w_res")):
        out += [(f"{a}.{n}.weight", (ct, ct), kind), (f"{a}.{n}.bias", (ct,), "b")]
    out += _vae_resnet("encoder.mid_block.resnets.1", ct, ct)
    out += [("encoder.conv_norm_out.weight", (ct,), "norm_w"), ("encoder.conv_norm_out.bias", (ct,), "norm_b"),
            ("encoder.conv_out.weight", (2 * cfg.latent_channels, ct, 3, 3), "w_mom"),
            ("encoder.conv_out.bias", (2 * cfg.latent_channels,), "b_mom"),
            ("quant_conv.weight", (8, 8, 1, 1), "w_q"), ("quant_conv.bias", (8,), "b")]
    return out


def num_vae_encoder_params(cfg: VAEConfig) -> int:
    return sum(math.prod(s) for _, s, _ in vae_encoder_param_specs(cfg))


def num_vae_decoder_params(cfg: VAEConfig) -> int:
    return sum(math.prod(s) for _, s, _ in vae_decoder_param_specs(cfg))


def synthetic_vae_state_dict(cfg: VAEConfig, seed: int = 4242, device="cpu", dtype=torch.float16,
                             with_encoder: bool = False) -> Dict[str, torch.Tensor]:
    """Seeded synthetic decoder (+ optionally encoder) weights with activation-preserving scales (same convention as
    weights.py). The decoder part does not depend on `with_encoder` (its draws come first)."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    specs = vae_decoder_param_specs(cfg) + (vae_encoder_param_specs(cfg) if with_encoder else [])
    for key, shape, kind in specs:
        if kind == "norm_w":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        elif kind in ("norm_b", "b"):
            t = 0.05 * torch.randn(shape, generator=g, device=device)
        elif kind == "w_pq":
            t = torch.eye(4, device=device).reshape(4, 4, 1, 1) + 0.1 * torch.randn(shape, generator=g, device=device)
        elif kind == "w_q":
            t = torch.eye(8, device=device).reshape(8, 8, 1, 1) + 0.1 * torch.randn(shape, generator=g, device=device)
        elif kind == "b_mom":   # mean rows ~ 0, log-variance rows ~ -3 (std ~ 0.2), as a trained posterior looks
            t = torch.cat([0.05 * torch.randn(shape[0] // 2, generator=g, device=device),
                           -3.0 + 0.3 * torch.randn(shape[0] // 2, generator=g, device=device)])
        else:
            fan_in = math.prod(shape[1:])
            gain = {"w": 1.0, "w_qk": 1.2, "w_res": 0.4, "w_out": 1.0, "w_mom": 1.0}[kind]
            t = torch.randn(shape, generator=g, device=device) * (gain / math.sqrt(fan_in))
        sd[key] = t.to(dtype)
    return sd


class NativeVAEDecoder(nv.NativeHandle):
    """Owner of one `cfgpp_vae_handle`. `decode(zt)` has the contract of the reference's `SDXL.decode` /
    `StableDiffusion.decode`: it takes the SCALED latent and returns `vae.decode(zt / scaling_factor).sample.float()`."""

    _prefix, _what = "_vae", "VAE decoder"

    def __init__(self, cfg: VAEConfig, state_dict: Dict[str, torch.Tensor], device="cuda:0"):
        self.cfg = cfg
        self.has_encoder = "encoder.conv_in.weight" in state_dict
        specs = vae_decoder_param_specs(cfg) + (vae_encoder_param_specs(cfg) if self.has_encoder else [])

        def weights():
            for key, _, _ in specs:
                if key not in state_dict:
                    raise KeyError(f"VAE state dict lacks '{key}'")
                w = state_dict[key]
                yield key, (w if w.dtype in (torch.float16, torch.float32) else w.float())

        self._open(to_vae_desc(cfg), weights(), device)

    @property
    def scale_factor(self) -> int:
        return 2 ** (len(self.cfg.block_out_channels) - 1)

    def decode_fp16(self, zt: torch.Tensor) -> torch.Tensor:
        assert zt.dim() == 4 and zt.shape[1] == 4, "latent must be (B,4,h,w)"
        zt = zt.detach().to(self.device)
        if zt.dtype not in (torch.float16, torch.float32):
            zt = zt.float()
        zt = zt.contiguous()
        b, _, h, w = zt.shape
        s = self.scale_factor
        img = torch.empty((b, self.cfg.out_channels, s * h, s * w), dtype=torch.float16, device=self.device)
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_vae_decode(self._h, nv.ptr(zt), c_int(0 if zt.dtype == torch.float16 else 1), c_int(b),
                                               c_int(h), c_int(w), nv.ptr(img), nv.stream_ptr()))
        return img

    def decode(self, zt: torch.Tensor) -> torch.Tensor:
        return self.decode_fp16(zt).float()

    def encode(self, x: torch.Tensor, noise: torch.Tensor | None = None, sample: bool = True) -> torch.Tensor:
        """`vae.encode(x).latent_dist.sample() * scaling_factor` (latent_sdxl.py:151-152, latent_diffusion.py:117-121):
        x (B,3,H,W) in [-1, 1] -> fp32 latent (B,4,H/f,W/f) (the fp16 module under the reference's autocast returns
        fp32: `exp` promotes the posterior's std). `noise`: the posterior's N(0,1) draw; when omitted it is
        drawn here with `torch.randn(mean.shape, dtype=fp16, device=cuda)` — the call diffusers' `randn_tensor` makes.
        `sample=False` returns the scaled posterior mean."""
        if not self.has_encoder:
            raise nv.NativeError("this VAE handle was built without encoder weights (encoder.*, quant_conv.*)")
        assert x.dim() == 4 and x.shape[1] == 3, "image must be (B,3,H,W)"
        x = x.detach().to(self.device)
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        b, _, h, w = x.shape
        s = self.scale_factor
        if sample and noise is None:
            noise = torch.randn((b, 4, h // s, w // s), dtype=torch.float16, device=self.device)
        if noise is not None:
            noise = noise.detach().to(self.device, torch.float16).contiguous()
            assert tuple(noise.shape) == (b, 4, h // s, w // s), "noise must have the latent's shape"
        out = torch.empty((b, 4, h // s, w // s), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_vae_encode(self._h, nv.ptr(x), c_int(0 if x.dtype == torch.float16 else 1), c_int(b),
                                               c_int(h), c_int(w), nv.ptr(noise if sample else None), nv.ptr(out),
                                               nv.stream_ptr()))
        return out

    @property
    def stats(self) -> dict:
        f, ws = c_double(), c_size_t()
        nv.check(self.lib.cfgpp_vae_stats(self._h, byref(f), byref(ws)))
        return {"flops": f.value, "workspace_bytes": ws.value}


class NativeVAE:
    """What the solver classes hold as `self.vae`: `decode` and `encode` on the native AutoencoderKL (the stand-in
    of conditioning.py only when the handle was built from a decoder-only state dict)."""

    def __init__(self, decoder: NativeVAEDecoder):
        self.decoder = decoder
        self._enc = None if decoder.has_encoder else LatentPreviewDecoder(decoder.scale_factor)

    def decode(self, zt: torch.Tensor) -> torch.Tensor:
        return self.decoder.decode(zt)

    def encode(self, x: torch.Tensor, dtype=torch.float16) -> torch.Tensor:
        if self._enc is not None:
            return self._enc.encode(x, dtype)
        return self.decoder.encode(x)   # fp32, as the reference's autocast region yields (`dtype` only steers the stand-in)


_VAES: Dict[tuple, NativeVAE] = {}


def get_vae(kind: str, device, model_key: str = "synthetic:4242") -> NativeVAE:
    """Cached native VAE per (kind, device, weights). `model_key`: a diffusers-format AutoencoderKL `*.safetensors`
    path, or 'synthetic[:seed]' (nothing can be downloaded here)."""
    dev = torch.device(device)
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    key = (kind, idx, model_key)
    if key not in _VAES:
        cfg = VAE_CONFIGS[kind]()
        if model_key.endswith(".safetensors"):
            from safetensors.torch import load_file
            sd = {k: v for k, v in load_file(model_key).items()
                  if k.startswith(("decoder.", "post_quant_conv.", "encoder.", "quant_conv."))}
        else:
            seed = int(model_key.split(":", 1)[1]) if ":" in model_key else 4242
            sd = synthetic_vae_state_dict(cfg, seed=seed, device=torch.device("cuda", idx), with_encoder=True)
        _VAES[key] = NativeVAE(NativeVAEDecoder(cfg, sd, torch.device("cuda", idx)))
    return _VAES[key]


def release_vaes():
    for v in _VAES.values():
        v.decoder.close()
    _VAES.clear()


def warn_synthetic(what: str):
    warnings.warn(f"no VAE checkpoint for {what} is available offline; decoding with seeded synthetic VAE weights "
                  f"(pass vae=... or a *.safetensors path for real weights)")
