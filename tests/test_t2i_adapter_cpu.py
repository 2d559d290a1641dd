"""T2I-Adapter host logic without a GPU: config parsing and refusals, the key census against the oracle module, the
feature placements on every UNet at the production sizes and SDXL buckets, the adapter_conditioning_factor table, the
oracle UNet with zero features, and sample()'s argument checks."""
import json

import pytest
import torch

import controlnet_oracle as CO
import production as P
import t2i_adapter_oracle as TO
from cfgpp_b200 import config as C, t2i_adapter as T


def _diffusers_config(**kw):
    cfg = {"_class_name": "T2IAdapter", "adapter_type": "full_adapter", "channels": [320, 640, 1280, 1280],
           "downscale_factor": 8, "in_channels": 3, "num_res_blocks": 2}
    cfg.update(kw)
    return cfg


@pytest.mark.parametrize("kw,expect", [({}, ("full_adapter", 3, 8, 64)),
                                       ({"in_channels": 1}, ("full_adapter", 1, 8, 64)),
                                       ({"adapter_type": "full_adapter_xl", "downscale_factor": 16},
                                        ("full_adapter_xl", 3, 16, 32))])
def test_config_parsing(kw, expect):
    cfg = T.config_from_diffusers(_diffusers_config(**kw))
    assert (cfg.adapter_type, cfg.in_channels, cfg.downscale_factor, cfg.total_downscale_factor) == expect
    assert cfg.channels == (320, 640, 1280, 1280) and cfg.num_res_blocks == 2


@pytest.mark.parametrize("kw,match", [({"adapter_type": "light_adapter"}, "light_adapter"),
                                      ({"_class_name": "MultiAdapter"}, "MultiAdapter"),
                                      ({"in_channels": 4}, "in_channels"),
                                      ({"channels": [320, 640, 1280]}, "4 blocks")])
def test_config_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        T.config_from_diffusers(_diffusers_config(**kw))


def test_channels_that_do_not_match_the_base_unet_are_refused():
    sd15, sdxl = C.sd15_config(), C.sdxl_config()
    with pytest.raises(ValueError, match="T2I-Adapter"):
        T.check_placements(T.t2i_adapter_config(sd15), sdxl, 1024, 1024)
    with pytest.raises(ValueError, match="T2I-Adapter"):
        T.check_placements(T.T2IAdapterConfig(channels=(320, 640, 640, 1280)), sd15, 512, 512)
    with pytest.raises(ValueError, match="T2I-Adapter"):
        T.T2IAdapter("x", "cpu", base_cfg=sdxl, config=T.t2i_adapter_config(sd15))


def test_checkpoint_finder(tmp_path):
    from cfgpp_b200.checkpoints import find_t2i_adapter_files
    with pytest.raises(FileNotFoundError, match="T2I-Adapter directory is missing"):
        find_t2i_adapter_files(tmp_path)
    (tmp_path / "config.json").write_text(json.dumps(_diffusers_config()))
    (tmp_path / "diffusion_pytorch_model.safetensors").write_bytes(b"")
    f = find_t2i_adapter_files(tmp_path)
    assert f["config"].name == "config.json" and f["weights"].name == "diffusion_pytorch_model.safetensors"


@pytest.mark.parametrize("name,in_channels", [("sd15", 3), ("sd15", 1), ("sdxl", 3), ("sdxl", 1), ("tiny_sd15", 3),
                                              ("tiny_sdxl", 1)])
def test_state_dict_key_census(name, in_channels):
    cfg = T.t2i_adapter_config(C.CONFIGS[name](), in_channels)
    with torch.device("meta"):
        m = TO.T2IAdapterModel(cfg)
    want = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k: tuple(s) for k, s, _ in T.t2i_adapter_param_specs(cfg)} == want


def _placement_cases():
    cases = P.t2i_sizes()
    from test_gpu_aspect_buckets import SDXL_BUCKETS  # latent (h, w) of every SDXL aspect-ratio bucket
    cases += [("sdxl", h, w) for h, w in SDXL_BUCKETS]
    cases += [("tiny_sd15", 32, 32), ("tiny_sd15", 16, 32), ("tiny_sd2", 16, 16), ("tiny_sdxl", 32, 32),
              ("tiny_sdxl", 16, 24)]
    return cases


@pytest.mark.parametrize("name,h,w", _placement_cases())
def test_feature_shapes_equal_the_tensors_they_land_on(name, h, w):
    """The adapter's feature shapes against the UNet tensors they land on, derived from its block structure."""
    ucfg = C.CONFIGS[name]()
    acfg = T.t2i_adapter_config(ucfg)
    feats = acfg.feature_shapes(8 * h, 8 * w)
    T.check_placements(acfg, ucfg, 8 * h, 8 * w)
    places = T.unet_placements(ucfg, h, w)
    L = len(ucfg.block_out_channels)
    assert feats == places[:len(feats)] and len(feats) in (L, L + 1)
    assert (len(feats) == L + 1) == (ucfg.addition_embed_type == "text_time")


@pytest.mark.parametrize("n,factor", [(20, 1.0), (20, 0.5), (20, 0.0), (7, 0.33), (50, 0.8), (3, 0.999)])
def test_factor_table(n, factor):
    assert T.step_flags(n, factor) == [i < int(n * factor) for i in range(n)]


def test_factor_table_over_two_s_entries_and_refiner_splits():
    from cfgpp_b200 import controlnet as CN, kdiffusion as K, schedule as S
    sigmas = K.get_sigmas_karras(6, 0.03, 14.6, rho=7.)
    steps, _ = S.kd_ancestral_steps(sigmas, lambda s: torch.tensor(500), 0.6, True, two_s=True)
    idx = CN.entry_steps(steps)
    n = len(sigmas) - 1
    assert idx[-1] == n - 1 and len(steps) > n
    flags = T.entry_flags(steps, 0.5)
    assert flags == [i < int(n * 0.5) for i in idx]
    ddim = S.ddim_cfgpp_steps(S.Schedule.make(20), 0.6, sdxl_indexing=True)
    table = T.entry_flags(ddim, 0.3)
    assert table == [True] * 6 + [False] * 14
    req = T.T2IRequest([], 0.3)
    assert [req.step_on(i, 20) for i in range(20)] == table == req.entry_flags(ddim)


@pytest.mark.parametrize("name", ["tiny_sd15", "tiny_sdxl"])
def test_oracle_unet_with_zero_features_is_the_oracle_forward(name):
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
    zeros = [torch.zeros(2, c, h, w) for c, h, w in T.t2i_adapter_config(cfg).feature_shapes(128, 128)]
    with torch.no_grad():
        ref = m(z, 500, ctx, add)["sample"]
        assert torch.equal(TO.unet_forward(m, z, 500, ctx, add, zeros)["sample"], ref)
        assert torch.equal(TO.unet_forward(m, z, 500, ctx, add)["sample"], ref)
        ones = [torch.ones_like(f) for f in zeros]
        assert not torch.equal(TO.unet_forward(m, z, 500, ctx, add, ones)["sample"], ref)


class _FakeAdapter(T.T2IAdapter):
    def __init__(self, cfg):  # no device handle: the argument checks only read the config
        self.cfg, self.base_cfg = cfg, None

    def features(self, image, scale=1.0):
        return [torch.zeros(image.shape[0], h, w, c) for c, h, w in self.cfg.feature_shapes(*image.shape[2:])]


@pytest.mark.parametrize("kw,match", [({"t2i_adapter_image": torch.rand(1, 3, 512, 512)}, "go together"),
                                      ({"t2i_adapter": "ad"}, "go together"),
                                      ({"t2i_adapter": "ad", "t2i_adapter_image": torch.rand(1, 3, 256, 512)},
                                       "resized"),
                                      ({"t2i_adapter": "ad", "t2i_adapter_image": torch.rand(1, 1, 512, 512)},
                                       "channels"),
                                      ({"t2i_adapter": "ad", "t2i_adapter_image": torch.rand(3, 3, 512, 512)},
                                       "batch"),
                                      ({"t2i_adapter": "ad", "t2i_adapter_image": torch.rand(1, 3, 512, 512),
                                        "adapter_conditioning_factor": 1.5}, r"\[0, 1\]"),
                                      ({"t2i_adapter": "ad", "t2i_adapter_image": torch.rand(1, 3, 512, 512),
                                        "adapter_conditioning_factor": -0.1}, r"\[0, 1\]"),
                                      ({"t2i_adapter": "xl", "t2i_adapter_image": torch.rand(1, 3, 512, 512)},
                                       "T2I-Adapter"),
                                      ({"t2i_adapter": object(), "t2i_adapter_image": torch.rand(1, 3, 512, 512)},
                                       "takes a cfgpp_b200.t2i_adapter.T2IAdapter")])
def test_sample_arguments_are_validated(kw, match):
    sd15 = C.sd15_config()
    kw = dict(kw)
    if kw.get("t2i_adapter") == "ad":
        kw["t2i_adapter"] = _FakeAdapter(T.t2i_adapter_config(sd15))
    elif kw.get("t2i_adapter") == "xl":  # an SDXL adapter on an SD v1.5 UNet
        kw["t2i_adapter"] = _FakeAdapter(T.t2i_adapter_config(C.sdxl_config()))
    with pytest.raises(ValueError, match=match):
        T.t2i_request(kw, sd15, 2, 512, 512)
    assert T.t2i_request({}, sd15, 2, 512, 512) is None
    req = T.t2i_request({"t2i_adapter": _FakeAdapter(T.t2i_adapter_config(sd15)),
                         "t2i_adapter_image": torch.rand(1, 3, 512, 512), "adapter_conditioning_factor": 0.5},
                        sd15, 2, 512, 512)
    assert [f.shape[0] for f in req.features] == [2] * 4 and req.factor == 0.5


@pytest.mark.parametrize("family,name", [("sd", "ddim_inversion"), ("sd", "ddim_inversion_cfg++"), ("sd", "ddim_edit"),
                                         ("sd", "ddim_edit_cfg++"), ("sdxl", "ddim_edit"), ("sdxl", "ddim_edit_cfg++")])
def test_inversion_and_editing_solvers_refuse_a_t2i_adapter(family, name):
    from cfgpp_b200 import latent_diffusion as LD, latent_sdxl as LX
    cls = (LD if family == "sd" else LX).__SOLVER__[name]
    kw = dict(t2i_adapter=_FakeAdapter(T.t2i_adapter_config(C.sd15_config())),
              t2i_adapter_image=torch.rand(1, 3, 64, 64))
    with pytest.raises(ValueError, match="does not take a T2I-Adapter"):
        if family == "sd":
            cls.sample(None, None, **kw)
        else:
            cls.sample(None, **kw)
