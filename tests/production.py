"""The production sizes every per-element kernel pin derives its cases from, and the attention launches of a UNet.

`test_gpu_gemm.py`, `test_gpu_norms.py` and `test_gpu_attention.py` walk these tables through their derivation
functions; `test_production_lists_cpu.py` asserts that every full-size model, text tower, vision tower, ControlNet-capable
UNet, IP-Adapter (plain and Plus) and T2I-capable UNet is listed, so a model added without sizes fails on any
machine."""

# latent (h, w) per full-size UNet config of `config.CONFIGS`: the native resolution first, then the non-square sizes
# whose levels are not multiples of 64 tokens (1216x832: 76x52 = 3952 tokens at level 1, 19x13 at level 3;
# 1344x768: 21x12 at level 3)
UNET_SIZES = {
    "sdxl": ((128, 128), (152, 104)),
    "sd15": ((64, 64),),
    "sd2": ((96, 96), (96, 64)),
    "sd2_base": ((64, 64),),
    "sdxl_refiner": ((128, 128), (152, 104), (168, 96)),
}

# AutoencoderKL image (H, W): SDXL 1024² and the 1216x832 bucket, SD 2 768² and 768x512, SD v1.5 / SD 2-base 512²
VAE_SIZES = ((1024, 1024), (1216, 832), (768, 768), (768, 512), (512, 512))

# text towers of `text_encoder.CLIP_CONFIGS` and the prompt batches they run at (M = 77·B)
TEXT_TOWERS = {"clip_l": (1, 2, 8), "clip_bigg": (1, 2, 8), "clip_h": (1, 2, 8)}

# the UNets that take a ControlNet (every UNET_SIZES entry but the SDXL refiner, which refuses one) at the same latent
# sizes; the conditioning embedding runs at the image size (8x the latent) for 1 image and the engine's maximum of 8
CONTROLNET_SIZES = {
    "sdxl": ((128, 128), (152, 104)),
    "sd15": ((64, 64),),
    "sd2": ((96, 96), (96, 64)),
    "sd2_base": ((64, 64),),
}
CONTROL_IMAGE_BATCHES = (1, 8)

# IP-Adapters: (base UNet, image-embedding width E): SD v1.5 with ViT-H (1024), SDXL with the default ViT-bigG tower
# (1280) and the ViT-H adapters for SDXL (1024); each projects one image embedding to IP_TOKENS image tokens
IP_ADAPTERS = (("sd15", 1024), ("sdxl", 1280), ("sdxl", 1024))
IP_TOKENS = 4

# IP-Adapter Plus: (base UNet, ViT-H hidden width E); the Resampler (`ip_adapter.plus_geometry`) reads the tower's
# penultimate hidden states and gives num_queries = 16 image tokens. It runs at UNet batch NB = 2, 4 and 16 (1, 2 and
# 8 images with CFG)
IP_PLUS_ADAPTERS = (("sd15", 1280), ("sdxl", 1280))
IP_PLUS_NB = (2, 4, 16)

# T2I-Adapters: base UNet -> latent (h, w) (the adapter image is 8h x 8w), for every UNet a T2I-Adapter conditions
# (not the SDXL refiner: the refiner runs after the hand-off without features). The UNet's sizes, plus SD v1.5 at
# 512x768, whose adapter levels are 96/48/24/12 wide and take the im2col A tile; the adapter runs for 1 image and the
# engine's maximum of 8, on 3-channel and 1-channel (sketch, canny) images
T2I_ADAPTER_SIZES = {
    "sd15": ((64, 64), (64, 96)),
    "sd2": ((96, 96), (96, 64)),
    "sd2_base": ((64, 64),),
    "sdxl": ((128, 128), (152, 104)),
}
T2I_ADAPTER_BATCHES = (1, 8)
T2I_IN_CHANNELS = (3, 1)

# CLIP vision towers of `vision_encoder` (`<name>_config`) and the image batches they encode
VISION_TOWERS = {"vit_h": (1, 2, 8), "vit_bigg": (1, 2, 8)}

N_CTX = 77


def unet_sizes():
    """(model, h, w) over the table, in table order."""
    return [(m, h, w) for m, sizes in UNET_SIZES.items() for h, w in sizes]


def size_tag(model, h, w):
    """The case-id prefix of one (model, latent size): model and image width x height."""
    return f"{model}-{8 * w}x{8 * h}"


def unet_attn_launches(cfg, h, w, NB=4):
    """Every flash-attention launch of a UNet's body on an h x w latent at UNet batch NB, in `Unet::prepare` order:
    per transformer block the self-attention (heads, HW, HW, head_dim) and the cross-attention against the 77-token
    prompt (heads, HW, 77, head_dim), with the plan name and the algorithmic FLOPs 4·NB·heads·Nq·Nkv·head_dim."""
    ch, L, lpb = cfg.block_out_channels, len(cfg.block_out_channels), cfg.layers_per_block
    tl, nh = cfg.transformer_layers_per_block, cfg.num_attention_heads
    out = []

    def transformer(p, level):
        C, heads, H, W = ch[level], nh[level], h >> level, w >> level
        hd = C // heads
        for k in range(tl[level]):
            for attn, nkv in (("attn1", H * W), ("attn2", N_CTX)):
                out.append(dict(name=f"{p}.transformer_blocks.{k}.{attn}.sdpa", heads=heads, Nq=H * W, Nkv=nkv,
                                hd=hd, flops=4.0 * NB * heads * H * W * nkv * hd))

    for i in range(L):
        if cfg.down_block_types[i].startswith("CrossAttn"):
            for j in range(lpb):
                transformer(f"down_blocks.{i}.attentions.{j}", i)
    transformer("mid_block.attentions.0", L - 1)
    for i in range(L):
        if cfg.up_block_types[i].startswith("CrossAttn"):
            for j in range(lpb + 1):
                transformer(f"up_blocks.{i}.attentions.{j}", L - 1 - i)
    return out


def controlnet_sizes():
    """(model, h, w) over CONTROLNET_SIZES, in table order."""
    return [(m, h, w) for m, sizes in CONTROLNET_SIZES.items() for h, w in sizes]


def t2i_sizes():
    """(model, h, w) over T2I_ADAPTER_SIZES, in table order."""
    return [(m, h, w) for m, sizes in T2I_ADAPTER_SIZES.items() for h, w in sizes]


def vision_config(tower):
    from cfgpp_b200 import vision_encoder as V
    return getattr(V, f"{tower}_config")()
