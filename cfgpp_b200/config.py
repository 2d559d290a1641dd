"""UNet2DConditionModel structure descriptions (the diffusers `config.json` fields the hot path depends on).

Mirrors what the reference obtains implicitly through `pipe.unet.config` (latent_diffusion.py:67,
latent_sdxl.py:50-54). See SURVEY.md Appendix A.1.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Optional, Tuple

CFGPP_MAX_LEVELS = 4


@dataclass(frozen=True)
class UNetConfig:
    name: str
    sample_size: int
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",)
    up_block_types: Tuple[str, ...] = ("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3
    layers_per_block: int = 2
    transformer_layers_per_block: Tuple[int, ...] = (1, 1, 1, 1)
    num_attention_heads: Tuple[int, ...] = (8, 8, 8, 8)  # diffusers' `attention_head_dim` (a misnomer)
    cross_attention_dim: int = 768
    use_linear_projection: bool = False
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    addition_embed_type: Optional[str] = None
    addition_time_embed_dim: int = 256
    projection_class_embeddings_input_dim: int = 2816
    pooled_dim: int = 1280
    vae_scale_factor: int = 8
    prediction_type: str = "epsilon"  # scheduler_config.json: "epsilon" | "v_prediction" (SD 2.0-v / 2.1 at 768^2)

    @property
    def time_embed_dim(self) -> int:
        return self.block_out_channels[0] * 4

    @property
    def num_time_ids(self) -> int:
        """Time ids of the text_time add-embedding (6 for the SDXL base, 5 for the refiner), 0 without one. The native
        handle derives the same count from the same three fields and refuses one that does not divide."""
        if self.addition_embed_type != "text_time":
            return 0
        return (self.projection_class_embeddings_input_dim - self.pooled_dim) // self.addition_time_embed_dim


def sd15_config() -> UNetConfig:
    return UNetConfig(name="sd15", sample_size=64)


def sdxl_config() -> UNetConfig:
    return UNetConfig(
        name="sdxl", sample_size=128, block_out_channels=(320, 640, 1280),
        down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
        up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
        transformer_layers_per_block=(1, 2, 10), num_attention_heads=(5, 10, 20), cross_attention_dim=2048,
        use_linear_projection=True, addition_embed_type="text_time")


def tiny_sdxl_config(sample_size: int = 32) -> UNetConfig:
    """SDXL topology (text_time add-embedding, linear projections, head_dim 64) at test-sized widths."""
    return UNetConfig(
        name="tiny_sdxl", sample_size=sample_size, block_out_channels=(64, 128, 256),
        down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
        up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
        transformer_layers_per_block=(1, 1, 2), num_attention_heads=(1, 2, 4), cross_attention_dim=128,
        use_linear_projection=True, addition_embed_type="text_time", addition_time_embed_dim=32,
        projection_class_embeddings_input_dim=6 * 32 + 64, pooled_dim=64)


def sdxl_refiner_config() -> UNetConfig:
    """stabilityai/stable-diffusion-xl-refiner-1.0: 4 levels (384, 768, 1536, 1536) with attention on the middle two
    (4 transformer layers each and in the mid block, 64-wide heads), OpenCLIP bigG penultimate context only (1280), and
    a text_time add-embedding of 5 time ids: original size, crop top-left and an aesthetic score (2560 = 1280 + 5*256)."""
    return UNetConfig(
        name="sdxl_refiner", sample_size=128, block_out_channels=(384, 768, 1536, 1536),
        down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
        up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
        transformer_layers_per_block=(4, 4, 4, 4), num_attention_heads=(6, 12, 24, 24), cross_attention_dim=1280,
        use_linear_projection=True, addition_embed_type="text_time", projection_class_embeddings_input_dim=2560)


def tiny_sdxl_refiner_config(sample_size: int = 32) -> UNetConfig:
    """SDXL refiner topology (4 levels, attention on the middle two only, 5 time ids, head_dim 64) at test-sized
    widths. Its context is the hidden state of tiny_sdxl's second text tower (64 wide), as the refiner's is bigG's."""
    return UNetConfig(
        name="tiny_sdxl_refiner", sample_size=sample_size, block_out_channels=(64, 128, 256, 256),
        down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
        up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
        transformer_layers_per_block=(1, 1, 2, 2), num_attention_heads=(1, 2, 4, 4), cross_attention_dim=64,
        use_linear_projection=True, addition_embed_type="text_time", addition_time_embed_dim=32,
        projection_class_embeddings_input_dim=5 * 32 + 64, pooled_dim=64)


def tiny_sd15_config(sample_size: int = 32) -> UNetConfig:
    """SD v1.5 topology (4 levels, 1x1-conv projections, no add-embedding) at test-sized widths with head_dim 64."""
    return UNetConfig(name="tiny_sd15", sample_size=sample_size, block_out_channels=(64, 128, 256, 256),
                      num_attention_heads=(1, 2, 4, 4), cross_attention_dim=128)


def sd2_config(sample_size: int = 96, prediction_type: str = "v_prediction") -> UNetConfig:
    """stabilityai/stable-diffusion-2-1 (and 2.0-v): SD v1.5's 4 levels with linear projections, 64-wide heads
    (diffusers' `attention_head_dim` (5, 10, 20, 20)), OpenCLIP ViT-H context (1024), v-prediction at 768^2."""
    return UNetConfig(name="sd2" if prediction_type == "v_prediction" else "sd2_base", sample_size=sample_size,
                      num_attention_heads=(5, 10, 20, 20), cross_attention_dim=1024, use_linear_projection=True,
                      prediction_type=prediction_type)


def sd2_base_config() -> UNetConfig:
    """stabilityai/stable-diffusion-2-base (and 2.1-base): the SD 2 UNet at 512^2, epsilon prediction."""
    return sd2_config(sample_size=64, prediction_type="epsilon")


def tiny_sd2_config(sample_size: int = 32, prediction_type: str = "v_prediction") -> UNetConfig:
    """SD 2 topology (4 levels, linear projections, head_dim 64, v-prediction) at test-sized widths."""
    return UNetConfig(name="tiny_sd2", sample_size=sample_size, block_out_channels=(64, 128, 256, 256),
                      num_attention_heads=(1, 2, 4, 4), cross_attention_dim=128, use_linear_projection=True,
                      prediction_type=prediction_type)


CONFIGS = {"sd15": sd15_config, "sdxl": sdxl_config, "tiny_sdxl": tiny_sdxl_config, "tiny_sd15": tiny_sd15_config,
           "sd2": sd2_config, "sd2_base": sd2_base_config, "tiny_sd2": tiny_sd2_config,
           "sdxl_refiner": sdxl_refiner_config, "tiny_sdxl_refiner": tiny_sdxl_refiner_config}
PREDICTION_TYPES = {"epsilon": 0, "v_prediction": 1}


class ModelDescC(ctypes.Structure):
    """`cfgpp_model_desc` of include/cfgpp_b200.h."""
    _fields_ = [
        ("in_channels", ctypes.c_int), ("out_channels", ctypes.c_int), ("num_levels", ctypes.c_int),
        ("block_out_channels", ctypes.c_int * CFGPP_MAX_LEVELS), ("down_has_attn", ctypes.c_int * CFGPP_MAX_LEVELS),
        ("up_has_attn", ctypes.c_int * CFGPP_MAX_LEVELS), ("layers_per_block", ctypes.c_int),
        ("transformer_layers", ctypes.c_int * CFGPP_MAX_LEVELS), ("num_heads", ctypes.c_int * CFGPP_MAX_LEVELS),
        ("cross_attention_dim", ctypes.c_int), ("use_linear_projection", ctypes.c_int),
        ("norm_num_groups", ctypes.c_int), ("norm_eps", ctypes.c_float), ("addition_time_embed_dim", ctypes.c_int),
        ("projection_class_embeddings_input_dim", ctypes.c_int), ("pooled_dim", ctypes.c_int),
    ]


class ModelDescExC(ModelDescC):
    """The full `cfgpp_model_desc` (cfgpp_create_ex): ModelDescC, the layout cfgpp_create reads, + prediction_type."""
    _fields_ = [("prediction_type", ctypes.c_int)]


def to_desc(cfg: UNetConfig) -> ModelDescExC:
    if cfg.prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"unsupported prediction_type {cfg.prediction_type!r}")
    d = ModelDescExC()
    n = len(cfg.block_out_channels)
    d.in_channels, d.out_channels, d.num_levels = cfg.in_channels, cfg.out_channels, n
    for i in range(n):
        d.block_out_channels[i] = cfg.block_out_channels[i]
        d.down_has_attn[i] = int(cfg.down_block_types[i] == "CrossAttnDownBlock2D")
        d.up_has_attn[i] = int(cfg.up_block_types[i] == "CrossAttnUpBlock2D")
        d.transformer_layers[i] = cfg.transformer_layers_per_block[i]
        d.num_heads[i] = cfg.num_attention_heads[i]
    d.layers_per_block = cfg.layers_per_block
    d.cross_attention_dim = cfg.cross_attention_dim
    d.use_linear_projection = int(cfg.use_linear_projection)
    d.norm_num_groups = cfg.norm_num_groups
    d.norm_eps = cfg.norm_eps
    d.addition_time_embed_dim = cfg.addition_time_embed_dim if cfg.addition_embed_type == "text_time" else 0
    d.projection_class_embeddings_input_dim = cfg.projection_class_embeddings_input_dim
    d.pooled_dim = cfg.pooled_dim
    d.prediction_type = PREDICTION_TYPES[cfg.prediction_type]
    return d
