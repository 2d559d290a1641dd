"""Pure-PyTorch restatement of diffusers `ControlNetModel` / `ControlNetConditioningEmbedding` (guess_mode off) and of
`UNet2DConditionModel.forward` with `down_block_additional_residuals` / `mid_block_additional_residual`, for the
ControlNet parity tests. Built from oracle/unet.py's modules (TimestepEmbedding, DownBlock, MidBlock), so the blocks
are the ones the UNet tests already pin; the module attribute names are diffusers', so `state_dict()` keys are the
ControlNetModel keys. Test infrastructure only: never imported by the product path."""
from __future__ import annotations

import dataclasses

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import unet as O


class ControlNetConditioningEmbedding(nn.Module):
    def __init__(self, embedding_channels: int, channels, conditioning_channels: int = 3):
        super().__init__()
        self.conv_in = nn.Conv2d(conditioning_channels, channels[0], 3, padding=1)
        blocks = []
        for i in range(len(channels) - 1):
            blocks.append(nn.Conv2d(channels[i], channels[i], 3, padding=1))
            blocks.append(nn.Conv2d(channels[i], channels[i + 1], 3, padding=1, stride=2))
        self.blocks = nn.ModuleList(blocks)
        self.conv_out = nn.Conv2d(channels[-1], embedding_channels, 3, padding=1)

    def forward(self, conditioning):
        emb = F.silu(self.conv_in(conditioning))
        for blk in self.blocks:
            emb = F.silu(blk(emb))
        return self.conv_out(emb)


def _embeddings(m, cfg, sample, timestep, added_cond_kwargs):
    timesteps = timestep
    if not torch.is_tensor(timesteps):
        timesteps = torch.tensor([timesteps], dtype=torch.int64, device=sample.device)
    elif timesteps.dim() == 0:
        timesteps = timesteps[None].to(sample.device)
    timesteps = timesteps.expand(sample.shape[0])
    t_emb = O.get_timestep_embedding(timesteps, cfg.block_out_channels[0]).to(dtype=sample.dtype)
    emb = m.time_embedding(t_emb)
    if cfg.addition_embed_type == "text_time":
        text_embeds = added_cond_kwargs["text_embeds"]
        time_embeds = O.get_timestep_embedding(added_cond_kwargs["time_ids"].flatten(), cfg.addition_time_embed_dim)
        time_embeds = time_embeds.reshape((text_embeds.shape[0], -1))
        emb = emb + m.add_embedding(torch.concat([text_embeds, time_embeds], dim=-1).to(emb.dtype))
    return emb


class ControlNetModel(nn.Module):
    def __init__(self, cfg: O.UNetConfig, embedding_channels=(16, 32, 96, 256)):
        super().__init__()
        self.cfg = cfg
        boc = cfg.block_out_channels
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = O.TimestepEmbedding(boc[0], cfg.time_embed_dim)
        if cfg.addition_embed_type == "text_time":
            self.add_embedding = O.TimestepEmbedding(cfg.projection_class_embeddings_input_dim, cfg.time_embed_dim)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(boc[0], embedding_channels)
        down, zero = [], [nn.Conv2d(boc[0], boc[0], 1)]
        out_ch = boc[0]
        for i in range(len(boc)):
            in_ch, out_ch = out_ch, boc[i]
            final = i == len(boc) - 1
            down.append(O.DownBlock(cfg, i, in_ch, out_ch, is_final=final))
            zero += [nn.Conv2d(out_ch, out_ch, 1) for _ in range(cfg.layers_per_block + (0 if final else 1))]
        self.down_blocks = nn.ModuleList(down)
        self.controlnet_down_blocks = nn.ModuleList(zero)
        self.mid_block = O.MidBlock(cfg)
        self.controlnet_mid_block = nn.Conv2d(boc[-1], boc[-1], 1)

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale=1.0,
                added_cond_kwargs=None):
        """(down_block_res_samples, mid_block_res_sample), each scaled by conditioning_scale."""
        emb = _embeddings(self, self.cfg, sample, timestep, added_cond_kwargs)
        sample = self.conv_in(sample)
        sample = sample + self.controlnet_cond_embedding(controlnet_cond)
        down_res = (sample,)
        for blk in self.down_blocks:
            sample, res = blk(sample, emb, encoder_hidden_states)
            down_res += res
        sample = self.mid_block(sample, emb, encoder_hidden_states)
        down_res = [zc(r) for r, zc in zip(down_res, self.controlnet_down_blocks)]
        mid = self.controlnet_mid_block(sample)
        return [r * conditioning_scale for r in down_res], mid * conditioning_scale


def unet_forward(m: O.UNet2DConditionModel, sample, timestep, encoder_hidden_states, added_cond_kwargs=None,
                 down_block_additional_residuals=None, mid_block_additional_residual=None):
    """oracle/unet.py's UNet2DConditionModel.forward with diffusers' optional ControlNet residuals: each is added to
    its skip tensor (and to the mid-block output) after the down path and mid block have run. With both None it is
    the oracle's forward, op for op."""
    cfg = m.cfg
    emb = _embeddings(m, cfg, sample, timestep, added_cond_kwargs)
    sample = m.conv_in(sample)
    down_res = (sample,)
    for blk in m.down_blocks:
        sample, res = blk(sample, emb, encoder_hidden_states)
        down_res += res
    if down_block_additional_residuals is not None:
        down_res = tuple(r + a for r, a in zip(down_res, down_block_additional_residuals))
    sample = m.mid_block(sample, emb, encoder_hidden_states)
    if mid_block_additional_residual is not None:
        sample = sample + mid_block_additional_residual
    for blk in m.up_blocks:
        n = len(blk.resnets)
        res = down_res[-n:]
        down_res = down_res[:-n]
        sample, _ = blk(sample, res, emb, encoder_hidden_states)
    sample = m.conv_out(F.silu(m.conv_norm_out(sample)))
    return {"sample": sample}


def oracle_cfg(cfg):
    return O.UNetConfig(**{f.name: getattr(cfg, f.name) for f in dataclasses.fields(O.UNetConfig)})


def build_controlnet(cn_cfg, state_dict, dtype=torch.float32, device="cpu") -> ControlNetModel:
    """ControlNetModel for a cfgpp_b200.controlnet.ControlNetConfig, strictly loaded from `state_dict`."""
    with torch.device("meta"):
        m = ControlNetModel(oracle_cfg(cn_cfg.unet), cn_cfg.conditioning_embedding_out_channels)
    m.load_state_dict({k: v.to(device=device, dtype=dtype) for k, v in state_dict.items()}, strict=True, assign=True)
    return m.eval().requires_grad_(False)
