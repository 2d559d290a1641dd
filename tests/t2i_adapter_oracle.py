"""Pure-PyTorch restatement of diffusers 0.27.1 `T2IAdapter` (`FullAdapter`, `FullAdapterXL`, `AdapterBlock`,
`AdapterResnetBlock`) and of `UNet2DConditionModel.forward` with `down_intrablock_additional_residuals` (plus the
ControlNet residuals of controlnet_oracle.py), for the T2I-Adapter parity tests. Built from oracle/unet.py's modules;
the attribute names are diffusers', so `state_dict()` keys are the T2IAdapter keys. Test infrastructure only: never
imported by the product path."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

import controlnet_oracle as CO
from oracle import unet as O


class AdapterResnetBlock(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.block1 = nn.Conv2d(channels, channels, 3, padding=1)
        self.act = nn.ReLU()
        self.block2 = nn.Conv2d(channels, channels, 1)

    def forward(self, x):
        return self.block2(self.act(self.block1(x))) + x


class AdapterBlock(nn.Module):
    def __init__(self, cin: int, cout: int, num_res_blocks: int, down: bool = False):
        super().__init__()
        self.downsample = nn.AvgPool2d(2, 2, ceil_mode=True) if down else None
        self.in_conv = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self.resnets = nn.Sequential(*[AdapterResnetBlock(cout) for _ in range(num_res_blocks)])

    def forward(self, x):
        if self.downsample is not None:
            x = self.downsample(x)
        if self.in_conv is not None:
            x = self.in_conv(x)
        return self.resnets(x)


class Adapter(nn.Module):  # FullAdapter / FullAdapterXL
    def __init__(self, cfg):
        super().__init__()
        self.unshuffle = nn.PixelUnshuffle(cfg.downscale_factor)
        self.conv_in = nn.Conv2d(cfg.in_channels * cfg.downscale_factor ** 2, cfg.channels[0], 3, padding=1)
        self.body = nn.ModuleList([AdapterBlock(cin, cout, cfg.num_res_blocks, down)
                                   for cin, cout, down in cfg.blocks()])

    def forward(self, x):
        x = self.conv_in(self.unshuffle(x))
        features = []
        for block in self.body:
            x = block(x)
            features.append(x)
        return features


class T2IAdapterModel(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.adapter = Adapter(cfg)

    def forward(self, x):
        return self.adapter(x)


def build_t2i_adapter(cfg, state_dict, dtype=torch.float32, device="cpu") -> T2IAdapterModel:
    with torch.device("meta"):
        m = T2IAdapterModel(cfg)
    m.load_state_dict({k: v.to(device=device, dtype=dtype) for k, v in state_dict.items()}, strict=True, assign=True)
    return m.eval().requires_grad_(False)


def pipeline_features(m, image, scale, dtype=torch.float16):
    """What diffusers' adapter pipelines feed the UNet: the image cast to the adapter's dtype, each feature multiplied by
    the scale once, then repeated for both CFG halves."""
    return [torch.cat([f * scale] * 2) for f in m(image.to(dtype))]


def unet_forward(m: O.UNet2DConditionModel, sample, timestep, encoder_hidden_states, added_cond_kwargs=None,
                 down_intrablock_additional_residuals=None, down_block_additional_residuals=None,
                 mid_block_additional_residual=None):
    """controlnet_oracle.unet_forward with diffusers' T2I-Adapter features: feature k goes, in order, onto the last
    (resnet, attention) output of a CrossAttnDownBlock2D (before its downsampler) or onto a DownBlock2D's output (after
    its downsampler; in place, so the skip sees it), and a feature left over onto the mid-block output when the shapes
    match. The adapter's adds come before the ControlNet's. Without features it is controlnet_oracle's forward."""
    cfg = m.cfg
    emb = CO._embeddings(m, cfg, sample, timestep, added_cond_kwargs)
    sample = m.conv_in(sample)
    down_res = (sample,)
    feats = list(down_intrablock_additional_residuals or [])
    for blk in m.down_blocks:
        outputs = ()
        for j, resnet in enumerate(blk.resnets):
            sample = resnet(sample, emb)
            if blk.attentions is not None:
                sample = blk.attentions[j](sample, encoder_hidden_states)
                if j == len(blk.resnets) - 1 and feats:
                    sample = sample + feats.pop(0)
            outputs += (sample,)
        if blk.downsamplers is not None:
            sample = blk.downsamplers[0](sample)
            outputs += (sample,)
        if blk.attentions is None and feats:
            sample = sample + feats.pop(0)
            outputs = outputs[:-1] + (sample,)
        down_res += outputs
    if down_block_additional_residuals is not None:
        down_res = tuple(r + a for r, a in zip(down_res, down_block_additional_residuals))
    sample = m.mid_block(sample, emb, encoder_hidden_states)
    if feats and sample.shape == feats[0].shape:
        sample = sample + feats.pop(0)
    if mid_block_additional_residual is not None:
        sample = sample + mid_block_additional_residual
    for blk in m.up_blocks:
        n = len(blk.resnets)
        res = down_res[-n:]
        down_res = down_res[:-n]
        sample, _ = blk(sample, res, emb, encoder_hidden_states)
    sample = m.conv_out(F.silu(m.conv_norm_out(sample)))
    return {"sample": sample}
