"""CLIP text towers on the Blackwell-native backend (SURVEY.md §8 f3).

Replaces the reference's prompt conditioning: `self.text_encoder(ids)[0]` (SD v1.5, latent_diffusion.py:93-115) and
`text_enc(ids, output_hidden_states=True)` -> `hidden_states[-2]` / `[-(clip_skip + 2)]` plus output `[0]` for the two
SDXL encoders (latent_sdxl.py:77-128) — transformers `CLIPTextModel` (openai/clip-vit-large-patch14) and
`CLIPTextModelWithProjection` (OpenCLIP ViT-bigG) — through the C ABI (`cfgpp_clip_*`): the projection / MLP GEMMs on
the wgmma GEMM kernel, causal attention / embedding / activation kernels of csrc/text_kernels.cu. Weights use the
transformers key names (`text_model.*`, `text_projection.weight`); no checkpoint or vocabulary exists offline, so the
default solver path runs seeded synthetic weights behind the `HashTokenizer` stand-in (tokenizer.py) — pass
`*.safetensors` + vocab / merges paths for the real models. There is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import math
from ctypes import byref, c_double, c_float, c_int, c_size_t
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _native as nv
from .tokenizer import ClipBPETokenizer, EOS_TOKEN, HashTokenizer


@dataclass(frozen=True)
class CLIPTextConfig:
    name: str = "clip_l"
    vocab_size: int = 49408
    max_position_embeddings: int = 77
    hidden_size: int = 768
    intermediate_size: int = 3072
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    hidden_act: str = "quick_gelu"
    layer_norm_eps: float = 1e-5
    projection_dim: int = 0     # > 0: CLIPTextModelWithProjection
    eos_token_id: int = 2       # the SD / SDXL encoder configs keep the legacy value => arg-max pooling rule
    pad_token_id: int = 49407   # tokenizer side: CLIP-L pads with <|endoftext|>, the SDXL tokenizer_2 with "!" (id 0)


def clip_l_config() -> CLIPTextConfig:
    return CLIPTextConfig()


def clip_bigg_config() -> CLIPTextConfig:
    return CLIPTextConfig(name="clip_bigg", hidden_size=1280, intermediate_size=5120, num_hidden_layers=32,
                          num_attention_heads=20, hidden_act="gelu", projection_dim=1280, pad_token_id=0)


def clip_h_config() -> CLIPTextConfig:
    """OpenCLIP ViT-H/14 as SD 2.x's `CLIPTextModel` (text_encoder/config.json): 23 layers (the checkpoint drops the
    last of OpenCLIP's 24), gelu, conditioning on last_hidden_state; tokenizer pads with "!" (id 0)."""
    return CLIPTextConfig(name="clip_h", hidden_size=1024, intermediate_size=4096, num_hidden_layers=23,
                          num_attention_heads=16, hidden_act="gelu", pad_token_id=0)


def tiny_clip_config(projection_dim: int = 0, act: str = "quick_gelu") -> CLIPTextConfig:
    return CLIPTextConfig(name="tiny_clip" + ("_proj" if projection_dim else ""), vocab_size=256, hidden_size=128,
                          intermediate_size=256, num_hidden_layers=3, num_attention_heads=2, hidden_act=act,
                          projection_dim=projection_dim, pad_token_id=0 if projection_dim else 255)


CLIP_CONFIGS = {"clip_l": clip_l_config, "clip_bigg": clip_bigg_config, "clip_h": clip_h_config,
                "tiny_clip": tiny_clip_config}
_ACT = {"quick_gelu": 0, "gelu": 1}


class ClipDescC(ctypes.Structure):
    _fields_ = [("vocab_size", c_int), ("max_positions", c_int), ("hidden_size", c_int), ("intermediate_size", c_int),
                ("num_layers", c_int), ("num_heads", c_int), ("hidden_act", c_int), ("projection_dim", c_int),
                ("layer_norm_eps", c_float)]


def to_clip_desc(cfg: CLIPTextConfig) -> ClipDescC:
    if cfg.hidden_act not in _ACT:
        raise ValueError(f"unsupported hidden_act {cfg.hidden_act}")
    return ClipDescC(cfg.vocab_size, cfg.max_position_embeddings, cfg.hidden_size, cfg.intermediate_size,
                     cfg.num_hidden_layers, cfg.num_attention_heads, _ACT[cfg.hidden_act], cfg.projection_dim,
                     cfg.layer_norm_eps)


def clip_param_specs(cfg: CLIPTextConfig) -> List[Tuple[str, Tuple[int, ...], str]]:
    """(transformers key, shape, init kind) in state-dict order."""
    d, i = cfg.hidden_size, cfg.intermediate_size
    out = [("text_model.embeddings.token_embedding.weight", (cfg.vocab_size, d), "emb"),
           ("text_model.embeddings.position_embedding.weight", (cfg.max_position_embeddings, d), "pos")]
    for l in range(cfg.num_hidden_layers):
        p = f"text_model.encoder.layers.{l}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            out += [(p + f"self_attn.{n}.weight", (d, d), "w_res" if n == "out_proj" else "w"), (p + f"self_attn.{n}.bias", (d,), "b")]
        out += [(p + "layer_norm1.weight", (d,), "norm_w"), (p + "layer_norm1.bias", (d,), "norm_b"),
                (p + "mlp.fc1.weight", (i, d), "w"), (p + "mlp.fc1.bias", (i,), "b"),
                (p + "mlp.fc2.weight", (d, i), "w_res"), (p + "mlp.fc2.bias", (d,), "b"),
                (p + "layer_norm2.weight", (d,), "norm_w"), (p + "layer_norm2.bias", (d,), "norm_b")]
    out += [("text_model.final_layer_norm.weight", (d,), "norm_w"), ("text_model.final_layer_norm.bias", (d,), "norm_b")]
    if cfg.projection_dim:
        out.append(("text_projection.weight", (cfg.projection_dim, d), "w"))
    return out


def num_clip_params(cfg: CLIPTextConfig) -> int:
    return sum(math.prod(s) for _, s, _ in clip_param_specs(cfg))


def synthetic_clip_state_dict(cfg: CLIPTextConfig, seed: int = 777, device="cpu", dtype=torch.float16) -> Dict[str, torch.Tensor]:
    """Seeded synthetic text-tower weights (activation-preserving scales, residual branches damped by depth)."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    damp = 1.0 / math.sqrt(2.0 * cfg.num_hidden_layers)
    for key, shape, kind in clip_param_specs(cfg):
        if kind == "norm_w":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        elif kind in ("norm_b", "b"):
            t = 0.02 * torch.randn(shape, generator=g, device=device)
        elif kind == "emb":
            t = 0.5 * torch.randn(shape, generator=g, device=device)
        elif kind == "pos":
            t = 0.25 * torch.randn(shape, generator=g, device=device)
        else:
            gain = 1.0 if kind == "w" else 2.0 * damp
            t = torch.randn(shape, generator=g, device=device) * (gain / math.sqrt(shape[1]))
        sd[key] = t.to(dtype)
    return sd


class NativeCLIPTextEncoder(nv.NativeHandle):
    """Owner of one `cfgpp_clip_handle`. `encode(ids, skip)` returns (hidden_states[L - skip], last_hidden_state,
    pooled): the three tensors the reference reads from the transformers output object."""

    _prefix, _what = "_clip", "text encoder"

    def __init__(self, cfg: CLIPTextConfig, state_dict: Dict[str, torch.Tensor], device="cuda:0"):
        self.cfg = cfg

        def weights():
            for key, shape, _ in clip_param_specs(cfg):
                if key not in state_dict:
                    raise KeyError(f"CLIP text state dict lacks '{key}'")
                w = state_dict[key]
                if tuple(w.shape) != tuple(shape):
                    raise ValueError(f"{key}: shape {tuple(w.shape)} != {tuple(shape)}")
                yield key, (w if w.dtype in (torch.float16, torch.float32) else w.float())

        self._open(to_clip_desc(cfg), weights(), device)

    def pooled_index(self, ids: torch.Tensor) -> torch.Tensor:
        """transformers' pooling row (modeling_clip.CLIPTextTransformer.forward)."""
        i = ids.to(torch.int)
        if self.cfg.eos_token_id == 2:
            return i.argmax(dim=-1).to(torch.int32)
        return (i == self.cfg.eos_token_id).int().argmax(dim=-1).to(torch.int32)

    def encode(self, ids: torch.Tensor, skip: int = 1, want_hidden=True, want_last=True, want_pooled=True):
        assert ids.dim() == 2, "input_ids must be (batch, tokens)"
        b, t = ids.shape
        if int(ids.min()) < 0 or int(ids.max()) >= self.cfg.vocab_size:
            raise ValueError("token id outside the vocabulary")
        ids_dev = ids.to(device=self.device, dtype=torch.int32).contiguous()
        pidx = self.pooled_index(ids_dev).contiguous() if want_pooled else None
        d = self.cfg.hidden_size
        hidden = torch.empty((b, t, d), dtype=torch.float16, device=self.device) if want_hidden else None
        last = torch.empty((b, t, d), dtype=torch.float16, device=self.device) if want_last else None
        pooled = torch.empty((b, self.cfg.projection_dim or d), dtype=torch.float16, device=self.device) if want_pooled else None
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_clip_encode(self._h, nv.ptr(ids_dev), nv.ptr(pidx), c_int(b), c_int(t), c_int(skip),
                                                nv.ptr(hidden), nv.ptr(last), nv.ptr(pooled), nv.stream_ptr()))
        return hidden, last, pooled

    @property
    def stats(self) -> dict:
        f, ws = c_double(), c_size_t()
        nv.check(self.lib.cfgpp_clip_stats(self._h, byref(f), byref(ws)))
        return {"flops": f.value, "workspace_bytes": ws.value}


class ClipConditioner:
    """The callable the solver classes hold as `text_encoder` / `text_enc_1` / `text_enc_2`: prompt -> (hidden, pooled)
    with the reference's choice of outputs. `mode='sdxl'`: (hidden_states[-(clip_skip + 2)], output[0]) as
    `SDXL._text_embed` (latent_sdxl.py:77-93); `mode='sd15'`: (last_hidden_state, None) as
    `StableDiffusion.get_text_embed` (latent_diffusion.py:93-115)."""

    def __init__(self, encoder: NativeCLIPTextEncoder, tokenizer, mode: str = "sdxl"):
        assert mode in ("sdxl", "sd15")
        self.encoder, self.tokenizer, self.mode = encoder, tokenizer, mode

    def input_ids(self, prompt) -> torch.Tensor:
        return torch.tensor(self.tokenizer(prompt), dtype=torch.int32)

    def __call__(self, prompt, device=None, clip_skip: Optional[int] = None):
        ids = self.input_ids(prompt)
        if self.mode == "sd15":
            _, last, _ = self.encoder.encode(ids, skip=0, want_hidden=False, want_last=True, want_pooled=False)
            return last, None
        skip = 1 if clip_skip is None else clip_skip + 1
        proj = self.encoder.cfg.projection_dim > 0
        hidden, last, pooled = self.encoder.encode(ids, skip=skip, want_hidden=True, want_last=not proj, want_pooled=proj)
        return hidden, (pooled if proj else last)   # output[0]: text_embeds | last_hidden_state

    def encode_batch(self, prompts: Sequence[str], clip_skip: Optional[int] = None, chunk: int = 16):
        """Many prompts per call (the 64-prompt runs of examples/text_to_mscoco.py): one native encode per `chunk`
        prompts instead of one per prompt; row i equals `self(prompts[i])`."""
        hs, ps = [], []
        for i in range(0, len(prompts), chunk):
            h, p = self(list(prompts[i:i + chunk]), clip_skip=clip_skip)
            hs.append(h)
            ps.append(p)
        return torch.cat(hs), (torch.cat(ps) if ps and ps[0] is not None else None)


_ENCODERS: Dict[tuple, NativeCLIPTextEncoder] = {}


def get_text_encoder(kind: str, device, model_key: str = "synthetic:777", cfg: Optional[CLIPTextConfig] = None
                     ) -> NativeCLIPTextEncoder:
    """Cached native text tower per (kind, device, weights). `model_key`: a transformers-format `*.safetensors` path or
    'synthetic[:seed]' (nothing can be downloaded here)."""
    dev = torch.device(device)
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    cfg = cfg or CLIP_CONFIGS[kind]()
    key = (cfg, idx, model_key)
    if key not in _ENCODERS:
        if model_key.endswith(".safetensors"):
            from safetensors.torch import load_file
            sd = load_file(model_key)
        else:
            seed = int(model_key.split(":", 1)[1]) if ":" in model_key else 777
            sd = synthetic_clip_state_dict(cfg, seed=seed, device=torch.device("cuda", idx))
        _ENCODERS[key] = NativeCLIPTextEncoder(cfg, sd, torch.device("cuda", idx))
    return _ENCODERS[key]


def get_conditioner(kind: str, device, mode: str, model_key: str = "synthetic:777", vocab_file: Optional[str] = None,
                    merges_file: Optional[str] = None, cfg: Optional[CLIPTextConfig] = None) -> ClipConditioner:
    enc = get_text_encoder(kind, device, model_key, cfg)
    c = enc.cfg
    if vocab_file and merges_file:
        tok = ClipBPETokenizer(vocab_file, merges_file, pad_token=EOS_TOKEN if c.pad_token_id != 0 else "!")
    else:
        tok = HashTokenizer(c.vocab_size, c.pad_token_id)
    return ClipConditioner(enc, tok, mode)


def release_text_encoders():
    for e in _ENCODERS.values():
        e.close()
    _ENCODERS.clear()
