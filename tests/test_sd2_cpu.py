"""Stable Diffusion 2.x on the host side: parameter-count pins of the SD 2 UNet and the OpenCLIP ViT-H text tower, the
v-prediction rule (a Dirac-data known answer through the oracle's v path in fp64, k-diffusion's VDenoiser, the step
tables' (a, b) against the seams' own), `--model sd20` and the SD 2 pipeline-directory reader. No GPU."""
import json
import math
from types import SimpleNamespace

import pytest
import torch


def test_sd2_unet_parameter_count():
    from cfgpp_b200 import config as C, weights as Wt
    from oracle import sd2 as OV, unet as O
    with torch.device("meta"):
        m = O.UNet2DConditionModel(OV.sd2_config())
    assert O.count_params(m) == 865_910_724
    assert sum(math.prod(s) for _, s, _ in Wt.unet_param_specs(C.sd2_config())) == 865_910_724
    # -base is the same network at 512^2
    assert Wt.unet_param_specs(C.sd2_base_config()) == Wt.unet_param_specs(C.sd2_config())


def test_clip_h_parameter_count_matches_transformers():
    import transformers
    from cfgpp_b200 import text_encoder as TE
    cfg = TE.clip_h_config()
    tc = transformers.CLIPTextConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size,
                                     intermediate_size=cfg.intermediate_size, num_hidden_layers=cfg.num_hidden_layers,
                                     num_attention_heads=cfg.num_attention_heads, hidden_act=cfg.hidden_act,
                                     max_position_embeddings=cfg.max_position_embeddings,
                                     layer_norm_eps=cfg.layer_norm_eps)
    with torch.device("meta"):
        model = transformers.CLIPTextModel(tc)
    n = sum(p.numel() for p in model.parameters())
    assert n == 340_387_840 and TE.num_clip_params(cfg) == n
    assert {k for k, _, _ in TE.clip_param_specs(cfg)} == set(model.state_dict()) - {"text_model.embeddings.position_ids"}


def test_sd2_configs():
    from cfgpp_b200 import config as C
    v, base, tiny = C.sd2_config(), C.sd2_base_config(), C.tiny_sd2_config()
    assert (v.sample_size, v.prediction_type) == (96, "v_prediction")
    assert (base.sample_size, base.prediction_type) == (64, "epsilon")
    for cfg in (v, base, tiny):
        assert len(cfg.block_out_channels) == 4 and cfg.use_linear_projection
        assert all(c // h == 64 for c, h in zip(cfg.block_out_channels, cfg.num_attention_heads))
    assert C.to_desc(v).prediction_type == 1 and C.to_desc(base).prediction_type == 0
    assert C.to_desc(C.sd15_config()).prediction_type == 0
    # the desc cfgpp_create_ex reads = the cfgpp_create layout + one int
    import ctypes
    assert ctypes.sizeof(C.ModelDescExC) == ctypes.sizeof(C.ModelDescC) + 4
    with pytest.raises(ValueError):
        C.to_desc(C.sd2_config(prediction_type="sample"))


# ---- the v-prediction rule ----------------------------------------------------------------------------------------

class DiracV:
    """Exact v-model of data concentrated at one point x0: at level abar the posterior is x0 itself, so
    eps = (x_in - sqrt(abar) x0) / sqrt(1 - abar) and v = sqrt(abar) eps - sqrt(1 - abar) x0. `abar_of(t)` is the
    level the model associates with timestep t."""

    def __init__(self, x0, abar_of):
        self.x0, self.abar_of, self.calls = x0, abar_of, 0

    def __call__(self, z_in, t, encoder_hidden_states=None, added_cond_kwargs=None):
        self.calls += 1
        ab = torch.tensor(float(self.abar_of(int(t.reshape(-1)[0]))), dtype=torch.float64)
        x0 = torch.cat([self.x0] * (z_in.shape[0] // self.x0.shape[0]))
        eps = (z_in - ab.sqrt() * x0) / (1 - ab).sqrt()
        return {"sample": ab.sqrt() * eps - (1 - ab).sqrt() * x0}


def _dirac_inputs():
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    zT = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    uc, c = torch.zeros(2, 77, 8, dtype=torch.float64), torch.ones(2, 77, 8, dtype=torch.float64)
    return x0, zT, uc, c


@pytest.mark.parametrize("method", ["ddim", "ddim_cfg++"])
def test_dirac_known_answer_ddim_family(method):
    """Every deterministic DDIM-family sampler, fed the exact v of Dirac data through the oracle's v rule, lands on x0
    from any zT: the rule must invert the v-parameterisation at the sampler's own alpha(t)."""
    from oracle import samplers as OSm, schedule as OS, sd2 as OV
    x0, zT, uc, c = _dirac_inputs()
    tb = OS.make_tables(10)
    model = DiracV(x0, lambda t: OSm._alpha_sd15(tb, t))
    unet = OV.VPredUNet(model, OV.ddim_v_levels(tb))
    if method == "ddim":
        z0 = OSm.ddim_plain(unet, tb, zT, uc, c, 3.0)
        err = (z0 - x0).abs().max().item()
    else:
        seen = []  # the Tweedie estimate of EVERY step is x0 (each step's level is pinned, not only the last one's)
        z0 = OSm.sd15_ddim_cfgpp(unet, tb, zT, uc, c, 0.6, callback_fn=lambda i, t, kw: seen.append(kw["z0t"]) or kw)
        assert len(seen) == len(tb.timesteps)
        err = max((z - x0).abs().max().item() for z in seen)
    print(f"Dirac {method}: max |z0 - x0*| = {err:.2e} after {unet.calls} UNet calls")
    assert unet.calls == len(tb.timesteps) and err < 1e-5


@pytest.mark.parametrize("method", ["euler", "euler_cfg++", "dpm++_2m", "dpm++_2m_cfg++"])
def test_dirac_known_answer_ve_family(method):
    """The same known answer through the VE-cast loops: abar = 1 / (1 + sigma^2) at each call's sigma."""
    from oracle import samplers as OSm, schedule as OS, sd2 as OV
    x0, zT, uc, c = _dirac_inputs()
    tb = OS.make_tables(10)
    sigmas = OSm.karras_sigmas(tb).double()
    sig32 = OSm.karras_sigmas(tb)
    t_to_sigma = {int(OSm.kd_timestep(tb, s)): float(s) for s in sig32[:-1]}
    assert len(t_to_sigma) == len(sig32) - 1  # every call has its own timestep: the model can tell the level
    model = DiracV(x0, lambda t: 1.0 / (1.0 + t_to_sigma[t] ** 2))
    unet = OV.VPredUNet(model, OV.kd_v_levels(sig32))
    x = zT * (sigmas[0] ** 2 + 1) ** 0.5
    plus = method.endswith("cfg++")
    if method.startswith("euler"):
        den, x = OSm.kd_euler_cfgpp(unet, tb, x, sig32, uc, c, 0.6 if plus else 3.0, plus=plus)
    else:
        den, x = OSm.kd_dpmpp_2m_cfgpp_sd15(unet, tb, x, sig32, uc, c, 0.6 if plus else 3.0, plus=plus)
    err = max((den - x0).abs().max().item(), (x - x0).abs().max().item())
    print(f"Dirac {method}: max |x - x0*| = {err:.2e} after {unet.calls} UNet calls")
    assert unet.calls == len(sig32) - 1 and err < 1e-4


def test_dirac_known_answer_catches_a_wrong_level():
    """The known answer is sharp: converting with the previous step's level (an off-by-one) or with the sign of v
    flipped misses x0 by far more than rounding."""
    from oracle import samplers as OSm, schedule as OS, sd2 as OV
    x0, zT, uc, c = _dirac_inputs()
    tb = OS.make_tables(10)
    lv = OV.ddim_v_levels(tb)
    shifted = lv[:1] + lv[:-1]
    flipped = [(-a, b) for a, b in lv]
    for levels in (shifted, flipped):
        unet = OV.VPredUNet(DiracV(x0, lambda t: OSm._alpha_sd15(tb, t)), levels)
        z0 = OSm.sd15_ddim_cfgpp(unet, tb, zT, uc, c, 0.6)
        assert (z0 - x0).abs().max().item() > 1e-2


def test_ve_conversion_is_vdenoiser():
    """eps = a v + b (c_in x) with (a, b) = ve_v_coefs(sigma) gives k-diffusion's VDenoiser estimate
    x c_skip + v c_out (sigma_data = 1) through the VE Tweedie step x - sigma eps, in fp64."""
    from cfgpp_b200 import schedule as S
    from oracle import sd2 as OV
    g = torch.Generator().manual_seed(11)
    for sigma in (0.0292, 0.5, 1.0, 3.7, 14.6146):
        s = torch.tensor(sigma, dtype=torch.float64)
        x = torch.randn(64, generator=g, dtype=torch.float64) * (1 + sigma)
        v = torch.randn(64, generator=g, dtype=torch.float64)
        c_skip, c_out, c_in = 1 / (s ** 2 + 1), -s / (s ** 2 + 1) ** 0.5, 1 / (s ** 2 + 1) ** 0.5
        ref = x * c_skip + v * c_out
        for a, b in (S.ve_v_coefs(s), OV.ve_v_level(s)):
            eps = a * v + b * (c_in * x)
            assert torch.allclose(x - s * eps, ref, rtol=1e-12, atol=1e-12), sigma


def test_step_tables_carry_the_seams_coefficients():
    """The (a, b) the fused step reads per entry equal, bit for bit, what the un-fused seams use: alpha(t) of the
    DDIM loop (predict_noise), alpha(t - skip) for inversion, ve_v_coefs(sigma) of every VE call (_k_denoise) —
    including both calls of a DPM-Solver++(2S) step. Epsilon tables are untouched by it."""
    import numpy as np
    from cfgpp_b200 import kdiffusion as K, schedule as S
    f32 = lambda x: np.float32(float(x))  # noqa: E731
    sch = S.Schedule.make(12)
    steps = S.ddim_cfgpp_steps(sch, 0.6, sdxl_indexing=False)
    before = bytes(S.to_c_array(steps))
    ab = S.v_pred_coefs(S.STEP_DDIM_CFGPP, steps)
    assert bytes(S.to_c_array(steps)) == before
    for (a, b), t in zip(ab, sch.timesteps):
        at = sch.alpha(t)
        assert (a, b) == (f32(at.sqrt()), f32((1 - at).sqrt()))
    inv = S.ddim_inversion_cfgpp_steps(sch, 0.6)
    for (a, b), t in zip(S.v_pred_coefs(S.STEP_DDIM_INV_CFGPP, inv), reversed(sch.timesteps)):
        ap = sch.alpha(t - sch.skip)
        assert (a, b) == (f32(ap.sqrt()), f32((1 - ap).sqrt()))
    sigmas = K.get_sigmas_karras(8, 0.0292, 14.6146, rho=7.)
    ts = lambda s: torch.tensor(500)  # noqa: E731
    kd = S.kd_steps(sigmas, ts, 0.6, True, second_order=True, diff_guided=True)
    for (a, b), s in zip(S.v_pred_coefs(S.STEP_DPMPP2M_CFGPP, kd), sigmas[:-1]):
        ra, rb = S.ve_v_coefs(s)
        assert (a, b) == (f32(ra), f32(rb))
    two, _ = S.kd_ancestral_steps(sigmas, ts, 0.6, True, two_s=True)
    from oracle import sd2 as OV
    call_sigmas = []
    for a, b in OV.kd_v_levels(sigmas, two_s=True):
        call_sigmas.append((f32(a), f32(b)))
    got = [tuple(r) for r in S.v_pred_coefs(S.STEP_DPMPP2M_CFGPP, two)]
    assert got == call_sigmas and len(got) > len(sigmas) - 1


def test_torch_v_to_eps_rounding():
    """The product's torch form (used by the seams) is two fp32 products and an fp32 sum, rounded once to fp16."""
    from cfgpp_b200 import schedule as S
    g = torch.Generator().manual_seed(2)
    v = (torch.randn(4096, generator=g) * 3).half()
    x = (torch.randn(4096, generator=g) * 3).half()
    a, b = torch.tensor(0.8, dtype=torch.float32), torch.tensor(0.6, dtype=torch.float32)
    got = S.v_to_eps(v, x, a, b)
    ref = (v.double() * a.double()).float().double() + (x.double() * b.double()).float().double()
    ref = ref.float().half()
    assert got.dtype == torch.float16 and torch.equal(got, ref)


# ---- model plumbing ---------------------------------------------------------------------------------------------

def test_model_sd20_builds_an_sd2_solver(monkeypatch):
    """`--model sd20` goes to the SD registry with the SD 2 UNet config (not SD v1.5's, not the SDXL registry)."""
    import examples.text_to_img as T
    from cfgpp_b200 import config as C
    seen = {}

    def fake(registry):
        def get(method, **kw):
            seen.update(kw, registry=registry, method=method)
            return SimpleNamespace(cfg=kw.get("unet_config"))
        return get
    monkeypatch.setattr(T, "get_solver", fake("sd"))
    monkeypatch.setattr(T, "get_solver_sdxl", fake("sdxl"))
    s = T.build_solver("sd20", "ddim_cfg++", SimpleNamespace(num_sampling=5), "cpu")
    assert seen["registry"] == "sd" and s.cfg == C.sd2_config() and s.cfg.sample_size * 8 == 768
    seen.clear()
    T.build_solver("sd15", "ddim_cfg++", SimpleNamespace(num_sampling=5), "cpu")
    assert seen["registry"] == "sd" and "unet_config" not in seen
    seen.clear()
    T.build_solver("sdxl_lightning", "ddim_cfg++_lightning", SimpleNamespace(num_sampling=5), "cpu")
    assert seen["registry"] == "sdxl"
    assert T.model_family("sd20") == "sd20"


def _sd2_skeleton(root, prediction_type, sample_size):
    for d, name in (("unet", "diffusion_pytorch_model.fp16.safetensors"), ("vae", "diffusion_pytorch_model.safetensors"),
                    ("text_encoder", "model.safetensors")):
        (root / d).mkdir(parents=True)
        (root / d / name).write_bytes(b"")
    (root / "tokenizer").mkdir()
    (root / "tokenizer" / "vocab.json").write_text("{}")
    (root / "tokenizer" / "merges.txt").write_text("#version: 0.2\n")
    (root / "scheduler").mkdir()
    (root / "scheduler" / "scheduler_config.json").write_text(json.dumps(
        {"_class_name": "DDIMScheduler", "prediction_type": prediction_type, "steps_offset": 1}))
    (root / "unet" / "config.json").write_text(json.dumps({"sample_size": sample_size, "cross_attention_dim": 1024}))


@pytest.mark.parametrize("prediction_type,sample_size", [("v_prediction", 96), ("epsilon", 64)])
def test_sd2_pipeline_directory(tmp_path, monkeypatch, prediction_type, sample_size):
    """stable-diffusion-2-1 (768^2 v) and stable-diffusion-2-base (512^2 epsilon) directories: the SD v1.5 layout, the
    ViT-H text tower, and the UNet config taken from scheduler_config.json / unet/config.json."""
    from cfgpp_b200 import checkpoints as CK, config as C, text_encoder as TE, vae as V
    _sd2_skeleton(tmp_path, prediction_type, sample_size)
    f = CK.find_pipeline_files(tmp_path, "sd20")
    assert {"unet", "vae", "text_encoder", "scheduler_config", "unet_config"} <= set(f)
    calls = []
    monkeypatch.setattr(TE, "get_conditioner", lambda kind, *a, **k: calls.append(("te", kind)) or kind)
    monkeypatch.setattr(V, "get_vae", lambda kind, *a, **k: calls.append(("vae", kind)) or kind)
    kw = CK.solver_components(tmp_path, "sd20", "cpu")
    assert kw["unet_config"] == C.sd2_config(sample_size=sample_size, prediction_type=prediction_type)
    assert ("te", "clip_h") in calls and ("vae", "sd15_vae") in calls
    assert kw["model_key"].endswith(".fp16.safetensors")
    # without the optional config files: the 768^2 v-prediction model
    (tmp_path / "scheduler" / "scheduler_config.json").unlink()
    (tmp_path / "unet" / "config.json").unlink()
    assert CK.sd2_unet_config(CK.find_pipeline_files(tmp_path, "sd20")) == C.sd2_config()
    # SD v1.5 directories are read as before
    assert "scheduler_config" not in CK.find_pipeline_files(tmp_path, "sd15")
