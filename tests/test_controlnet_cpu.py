"""ControlNet pieces that need no GPU: config parsing and its refusals, the checkpoint finder, the state-dict key census,
the conditioning-scale table, the residual-taking oracle UNet and the control-image validation."""
import json

import pytest
import torch

import controlnet_oracle as CO
from cfgpp_b200 import config as C
from cfgpp_b200 import controlnet as CN
from cfgpp_b200.checkpoints import find_controlnet_files

SD15_CONTROLNET = {  # lllyasviel/sd-controlnet-canny config.json (the fields that shape the model)
    "_class_name": "ControlNetModel", "attention_head_dim": 8, "block_out_channels": [320, 640, 1280, 1280],
    "conditioning_embedding_out_channels": [16, 32, 96, 256], "controlnet_conditioning_channel_order": "rgb",
    "cross_attention_dim": 768, "down_block_types": ["CrossAttnDownBlock2D"] * 3 + ["DownBlock2D"],
    "global_pool_conditions": False, "in_channels": 4, "layers_per_block": 2, "norm_eps": 1e-05,
    "norm_num_groups": 32, "use_linear_projection": False}
SDXL_CONTROLNET = {  # diffusers/controlnet-canny-sdxl-1.0 config.json
    "_class_name": "ControlNetModel", "addition_embed_type": "text_time", "addition_time_embed_dim": 256,
    "attention_head_dim": [5, 10, 20], "block_out_channels": [320, 640, 1280], "conditioning_channels": 3,
    "conditioning_embedding_out_channels": [16, 32, 96, 256], "controlnet_conditioning_channel_order": "rgb",
    "cross_attention_dim": 2048, "down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
    "global_pool_conditions": False, "in_channels": 4, "layers_per_block": 2,
    "projection_class_embeddings_input_dim": 2816, "transformer_layers_per_block": [1, 2, 10],
    "use_linear_projection": True}


def _same_down_mid(a: C.UNetConfig, b: C.UNetConfig):
    fields = ("block_out_channels", "down_block_types", "layers_per_block", "transformer_layers_per_block",
              "num_attention_heads", "cross_attention_dim", "use_linear_projection", "addition_embed_type")
    return all(getattr(a, f) == getattr(b, f) for f in fields)


def test_config_parsing_matches_the_base_unets():
    sd15 = CN.config_from_diffusers(SD15_CONTROLNET)
    assert _same_down_mid(sd15.unet, C.sd15_config()) and sd15.conditioning_embedding_out_channels == (16, 32, 96, 256)
    xl = CN.config_from_diffusers(SDXL_CONTROLNET)
    assert _same_down_mid(xl.unet, C.sdxl_config())
    assert xl.unet.pooled_dim == 1280 and xl.unet.num_time_ids == 6
    assert len(sd15.residual_channels) == 13 and len(xl.residual_channels) == 10  # 12 / 9 down + the mid block


@pytest.mark.parametrize("field,value,match", [("global_pool_conditions", True, "global_pool"),
                                               ("controlnet_conditioning_channel_order", "bgr", "rgb"),
                                               ("conditioning_channels", 1, "conditioning_channels")])
def test_config_refusals(field, value, match):
    with pytest.raises(ValueError, match=match):
        CN.config_from_diffusers({**SD15_CONTROLNET, field: value})


def test_checkpoint_finder(tmp_path):
    with pytest.raises(FileNotFoundError, match="config.json"):
        find_controlnet_files(tmp_path)
    (tmp_path / "config.json").write_text(json.dumps(SD15_CONTROLNET))
    with pytest.raises(FileNotFoundError, match="diffusion_pytorch_model"):
        find_controlnet_files(tmp_path)
    (tmp_path / "diffusion_pytorch_model.safetensors").write_bytes(b"")
    assert find_controlnet_files(tmp_path)["weights"].name == "diffusion_pytorch_model.safetensors"
    (tmp_path / "diffusion_pytorch_model.fp16.safetensors").write_bytes(b"")
    files = find_controlnet_files(tmp_path)
    assert files["weights"].name == "diffusion_pytorch_model.fp16.safetensors"
    assert files["config"] == tmp_path / "config.json"


@pytest.mark.parametrize("name", ["sd15", "sdxl", "sd2", "tiny_sd15", "tiny_sdxl"])
def test_state_dict_key_census(name):
    """The synthetic specs name exactly the parameters of the restated ControlNetModel, with its shapes."""
    cfg = CN.controlnet_config(C.CONFIGS[name]())
    with torch.device("meta"):
        m = CO.ControlNetModel(CO.oracle_cfg(cfg.unet), cfg.conditioning_embedding_out_channels)
    want = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    got = {k: s for k, s, _ in CN.controlnet_param_specs(cfg)}
    assert got == want
    n_down = sum(1 for k in got if k.startswith("controlnet_down_blocks.") and k.endswith(".weight"))
    assert n_down == len(cfg.residual_channels) - 1 == (12 if len(cfg.unet.block_out_channels) == 4 else 9)


def _diffusers_keep(i, n, start, end):
    return 1.0 - float(i / n < start or (i + 1) / n > end)


@pytest.mark.parametrize("n,scale,start,end", [(10, 1.0, 0.0, 1.0), (10, 0.7, 0.2, 0.8), (25, 1.5, 0.0, 0.5),
                                               (7, 0.5, 0.3, 1.0)])
def test_control_scale_table(n, scale, start, end):
    table = CN.control_scales(n, scale, start, end)
    assert table == [scale * _diffusers_keep(i, n, start, end) for i in range(n)]
    two_s = CN.control_scales(n, scale, start, end, entries_per_step=2)  # DPM-Solver++(2S): two entries per step
    assert two_s[0::2] == table and two_s[1::2] == table
    k = n // 2  # a refiner split: the base runs steps [0, k), the refiner the rest, indices over the whole schedule
    assert CN.control_scales(n, scale, start, end, count=k) + CN.control_scales(n, scale, start, end, first=k) == table


@pytest.mark.parametrize("name", ["tiny_sd15", "tiny_sdxl"])
def test_oracle_unet_without_residuals_is_the_oracle_forward(name):
    from cfgpp_b200 import weights as Wt
    from oracle import unet as O
    cfg = C.CONFIGS[name]()
    m = O.build_unet(CO.oracle_cfg(cfg), Wt.synthetic_state_dict(cfg, seed=5, dtype=torch.float32))
    g = torch.Generator().manual_seed(0)
    z = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=g)
    add = None
    if cfg.addition_embed_type:
        add = {"text_embeds": torch.randn(2, cfg.pooled_dim, generator=g),
               "time_ids": torch.tensor([[128., 128, 0, 0, 128, 128]] * 2)}
    with torch.no_grad():
        assert torch.equal(CO.unet_forward(m, z, 500, ctx, add)["sample"], m(z, 500, ctx, add)["sample"])


def test_control_image_validation():
    img = torch.rand(1, 3, 64, 96)
    assert CN.check_control_image(img, 4, 64, 96).shape == (4, 3, 64, 96)
    assert CN.check_control_image(torch.rand(4, 3, 64, 96), 4, 64, 96).shape == (4, 3, 64, 96)
    with pytest.raises(ValueError, match="resized"):
        CN.check_control_image(img, 1, 64, 64)
    with pytest.raises(ValueError, match="batch"):
        CN.check_control_image(torch.rand(2, 3, 64, 96), 4, 64, 96)
    with pytest.raises(ValueError, match=r"\(B, 3, H, W\)"):
        CN.check_control_image(torch.rand(1, 1, 64, 96), 1, 64, 96)


# ---- solver arguments and the scale table over real schedules ---------------------------------------------------------
def _two_s_steps(n=6):
    from cfgpp_b200 import kdiffusion as K, schedule as S
    sigmas = K.get_sigmas_karras(n, 0.03, 14.6, rho=7.)
    steps, _ = S.kd_ancestral_steps(sigmas, lambda s: torch.tensor(500), 0.6, True, two_s=True)
    return sigmas, steps


def test_entry_scales_follow_the_sampler_steps():
    from cfgpp_b200 import schedule as S
    ddim = S.ddim_cfgpp_steps(S.Schedule.make(10), 0.6, sdxl_indexing=False)
    assert CN.entry_steps(ddim) == list(range(10))
    assert CN.entry_scales(ddim, 0.7, 0.2, 0.8) == CN.control_scales(10, 0.7, 0.2, 0.8)
    sigmas, two_s = _two_s_steps()
    n = len(sigmas) - 1
    idx = CN.entry_steps(two_s)
    assert idx[-1] == n - 1 and len(two_s) > n  # two entries per step where the step has a midpoint
    per_step = CN.control_scales(n, 0.9, 0.1, 0.6)
    assert CN.entry_scales(two_s, 0.9, 0.1, 0.6) == [per_step[i] for i in idx]
    for a, b in zip(two_s, idx):
        if a.coef.second_order & S.KD_2S_FINAL:  # the final entry of a step shares its midpoint's scale
            assert b == idx[two_s.index(a) - 1]


def test_refiner_split_keeps_whole_schedule_indices():
    """The base engine runs entries [0, k) of one table computed over the whole schedule; the refiner none."""
    from cfgpp_b200 import schedule as S
    steps = S.ddim_cfgpp_steps(S.Schedule.make(20), 0.6, sdxl_indexing=True)
    req = CN.ControlRequest(engine=None, image=torch.zeros(1), scale=1.0, start=0.0, end=0.5)
    table = req.entry_scales(steps)
    assert table == [1.0] * 10 + [0.0] * 10
    assert [req.step_scale(i, 20) for i in range(20)] == table  # the un-fused loops' per-step value


class _FakeNative(CN.NativeControlNet):
    def __init__(self):  # no device handle: only the type matters to the argument checks
        self.attached_to = None


@pytest.mark.parametrize("kw,match", [({"control_image": torch.rand(1, 3, 64, 64)}, "without controlnet"),
                                      ({"controlnet": "cn"}, "needs control_image"),
                                      ({"controlnet": "cn", "control_image": torch.rand(1, 3, 32, 64)}, "resized"),
                                      ({"controlnet": "cn", "control_image": torch.rand(3, 3, 64, 64)}, "batch"),
                                      ({"controlnet": "cn", "control_image": torch.rand(1, 3, 64, 64),
                                        "control_guidance_start": 0.6, "control_guidance_end": 0.4}, "start"),
                                      ({"controlnet": object(), "control_image": torch.rand(1, 3, 64, 64)},
                                       "takes a cfgpp_b200.controlnet.ControlNet")])
def test_solver_control_arguments_are_validated(kw, match):
    kw = dict(kw)
    if kw.get("controlnet") == "cn":
        kw["controlnet"] = _FakeNative()
    with pytest.raises(ValueError, match=match):
        CN.control_request(kw, 2, 64, 64, "cpu")
    assert CN.control_request({}, 2, 64, 64, "cpu") is None
    req = CN.control_request({"controlnet": _FakeNative(), "control_image": torch.rand(1, 3, 64, 64),
                              "controlnet_conditioning_scale": 0.5}, 2, 64, 64, "cpu")
    assert req.image.shape == (2, 3, 64, 64) and req.scale == 0.5


@pytest.mark.parametrize("family,name", [("sd", "ddim_inversion"), ("sd", "ddim_inversion_cfg++"), ("sd", "ddim_edit"),
                                         ("sd", "ddim_edit_cfg++"), ("sdxl", "ddim_edit"), ("sdxl", "ddim_edit_cfg++")])
def test_inversion_and_editing_solvers_refuse_a_controlnet(family, name):
    from cfgpp_b200 import latent_diffusion as LD, latent_sdxl as LX
    cls = (LD if family == "sd" else LX).__SOLVER__[name]
    with pytest.raises(ValueError, match="does not take a ControlNet"):
        if family == "sd":
            cls.sample(None, None, controlnet=_FakeNative(), control_image=torch.rand(1, 3, 64, 64))
        else:
            cls.sample(None, controlnet=_FakeNative(), control_image=torch.rand(1, 3, 64, 64))


def test_controlled_call_resets_the_request():
    from cfgpp_b200.solver_base import SolverBase

    class Host(SolverBase):
        device = "cpu"

    h = Host()

    def boom():
        assert h._control is not None
        raise RuntimeError("x")
    with pytest.raises(RuntimeError):
        h._controlled({"controlnet": _FakeNative(), "control_image": torch.rand(1, 3, 64, 64)}, 1, 8, 8, boom)
    assert h._control is None
