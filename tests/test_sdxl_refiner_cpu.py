"""The SDXL refiner on the host side: parameter-count pins of the refiner UNet, the expert split of the schedule and of
the DPM++ step table, the oracle's split loops against the unsplit ones when both experts are one module, the
refiner's aesthetic-score time ids and the refiner pipeline-directory reader. No GPU."""
import math

import pytest
import torch


def test_refiner_parameter_count():
    from cfgpp_b200 import config as C, weights as Wt
    from helpers import oracle_cfg
    from oracle import sdxl_refiner as OR, unet as O
    with torch.device("meta"):
        m = O.UNet2DConditionModel(OR.sdxl_refiner_config())
    assert O.count_params(m) == 2_259_526_660
    assert sum(math.prod(s) for _, s, _ in Wt.unet_param_specs(C.sdxl_refiner_config())) == 2_259_526_660
    assert oracle_cfg(C.sdxl_refiner_config()) == OR.sdxl_refiner_config()
    tiny = C.tiny_sdxl_refiner_config()
    with torch.device("meta"):
        mt = O.UNet2DConditionModel(oracle_cfg(tiny))
    assert O.count_params(mt) == sum(math.prod(s) for _, s, _ in Wt.unet_param_specs(tiny))


def test_refiner_configs():
    from cfgpp_b200 import config as C
    ref, tiny = C.sdxl_refiner_config(), C.tiny_sdxl_refiner_config()
    assert C.CONFIGS["sdxl_refiner"] is C.sdxl_refiner_config and C.CONFIGS["tiny_sdxl_refiner"] is C.tiny_sdxl_refiner_config
    for cfg in (ref, tiny):
        assert cfg.num_time_ids == 5 and len(cfg.block_out_channels) == 4
        assert cfg.down_block_types[0] == cfg.down_block_types[3] == "DownBlock2D"
        assert cfg.up_block_types[0] == cfg.up_block_types[3] == "UpBlock2D"
        assert all(c // h == 64 for c, h in zip(cfg.block_out_channels, cfg.num_attention_heads))
    assert (ref.cross_attention_dim, ref.pooled_dim, ref.projection_class_embeddings_input_dim) == (1280, 1280, 2560)
    # the tiny refiner's context is the tiny base's second text tower (as the refiner's is bigG)
    assert tiny.cross_attention_dim == tiny.pooled_dim == C.tiny_sdxl_config().pooled_dim
    assert C.sdxl_config().num_time_ids == 6 and C.tiny_sdxl_config().num_time_ids == 6
    assert C.sd15_config().num_time_ids == 0 and C.sd2_config().num_time_ids == 0
    d = C.to_desc(ref)
    assert (d.addition_time_embed_dim, d.projection_class_embeddings_input_dim, d.pooled_dim) == (256, 2560, 1280)


# ---- the split ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nfe,end,k,base_ts,refiner_ts", [(50, 0.8, 40, (981, 201), (181, 1)),
                                                          (30, 0.8, 23, (958, 232), (199, 1))])
def test_ddim_split_index(nfe, end, k, base_ts, refiner_ts):
    from cfgpp_b200 import schedule as S
    from oracle import schedule as OS, sdxl_refiner as OR
    sch = S.Schedule.make(nfe)
    got = S.expert_split(sch.timesteps, end, nfe)
    assert got == k == OR.split_index(OS.make_tables(nfe).timesteps, end, nfe)
    assert (sch.timesteps[0].item(), sch.timesteps[k - 1].item()) == base_ts
    assert (sch.timesteps[k].item(), sch.timesteps[-1].item()) == refiner_ts


def test_dpmpp_split_index_and_table():
    from cfgpp_b200 import schedule as S
    sch = S.Schedule.make(25)
    n = len(sch.timesteps) - 1
    k = S.expert_split(sch.timesteps, 0.8, n)
    assert (n, k) == (24, 20)
    full, s0 = S.dpmpp_2m_cfgpp_steps(sch, 0.6)
    split, s1 = S.dpmpp_2m_cfgpp_steps(sch, 0.6, restart_at=k)
    assert torch.equal(s0, s1) and len(full) == len(split) == n
    assert (full[0].t, sch.timesteps[k].item(), split[k].t) == (960.0, 161, 160.0)
    assert n - k == 4
    for i, (a, b) in enumerate(zip(full, split)):
        if i != k:
            assert bytes(a) == bytes(b), f"entry {i} changed"
    # entry k: the first-order (i == 0) form — same t, input scale and c's, no 2nd-order coefficients
    a, b = full[k], split[k]
    assert a.coef.second_order == 1 and b.coef.second_order == 0
    assert (b.t, b.in_scale, b.coef.c0, b.coef.c1, b.coef.c2, b.coef.c3) == \
        (a.t, a.in_scale, a.coef.c0, a.coef.c1, a.coef.c2, a.coef.c3)
    assert (b.coef.d0, b.coef.d1, b.coef.d2, b.coef.d3) == (0.0, 0.0, 0.0, 0.0)


@pytest.mark.parametrize("end,n", [(0.0, 50), (1.0, 50), (-0.1, 50), (0.999, 50), (0.01, 50), (0.8, 1)])
def test_split_rejects(end, n):
    """denoising_end outside (0, 1), or a split that leaves either expert with no step (k = 0 or k = n)."""
    from cfgpp_b200 import schedule as S
    from oracle import sdxl_refiner as OR
    sch = S.Schedule.make(50)
    with pytest.raises(ValueError):
        S.expert_split(sch.timesteps, end, n)
    with pytest.raises(ValueError):
        OR.split_index(sch.timesteps, end, n)


# ---- the oracle split with one module as both experts -------------------------------------------------------------

def _tiny_sdxl_oracle(B=2, hw=16):
    from cfgpp_b200 import config as C, weights as Wt
    from helpers import make_inputs, oracle_cfg
    from oracle import unet as O
    cfg = C.tiny_sdxl_config()
    sd = Wt.synthetic_state_dict(cfg, seed=3, device="cpu")
    m = O.build_unet(oracle_cfg(cfg), sd, dtype=torch.float32)
    z, uc, c, add = make_inputs(cfg, B, hw, "cpu", seed=5)
    return m, z, uc.float(), c.float(), {k: v.float() for k, v in add.items()}


@pytest.mark.parametrize("loop", ["ddim_cfg++", "ddim"])
def test_oracle_ddim_split_same_module_is_unsplit(loop):
    from oracle import samplers as OSm, schedule as OS, sdxl_refiner as OR
    m, z, uc, c, add = _tiny_sdxl_oracle()
    tb = OS.make_tables(8)
    k = OR.split_index(tb.timesteps, 0.8, 8)
    cond = (uc, c, add)
    if loop == "ddim_cfg++":
        ref = OSm.sdxl_ddim_cfgpp(m, tb, z, uc, c, 0.6, add)
        got = OR.sdxl_ddim_cfgpp_split(m, m, tb, z, cond, cond, 0.6, k)
    else:
        ref = OSm.ddim_plain(m, tb, z, uc, c, 0.6, add, sdxl_indexing=True)
        got = OR.sdxl_ddim_split(m, m, tb, z, cond, cond, 0.6, k)
    assert k == 6 and torch.equal(got, ref)


def test_oracle_dpmpp_split_resets_history_at_k():
    from oracle import samplers as OSm, schedule as OS, sdxl_refiner as OR
    m32, z, uc, c, add = _tiny_sdxl_oracle()

    def m(z_in, t, **kw):  # the fp32 module on the loop's fp16 state
        return m32(z_in.float(), t, **kw)
    tb = OS.make_tables(12)
    n = len(tb.timesteps) - 1
    k = OR.split_index(tb.timesteps, 0.8, n)
    cond = (uc, c, add)
    rec_full, rec_split = [], []
    full = OSm.sdxl_dpmpp_2m_cfgpp(m, tb, z, uc, c, 0.6, add, record=rec_full)
    split = OR.sdxl_dpmpp_2m_cfgpp_split(m, m, tb, z, cond, cond, 0.6, k, record=rec_split)
    assert 1 <= k < n - 1
    # the base part is the unsplit loop
    for i in range(k + 1):
        for key in ("x", "noise_uc", "noise_c"):
            assert torch.equal(rec_full[i][key], rec_split[i][key]), (i, key)
    # step k is the first-order update of a fresh call, from the handed-over state
    alphas = tb.alphas_cumprod[tb.timesteps.int()]
    sigmas = (1 - alphas).sqrt() / alphas.sqrt()
    r = rec_split[k]
    assert r["old_denoised"] is None and rec_full[k]["old_denoised"] is not None
    noise_pred = r["noise_uc"] + 0.6 * (r["noise_c"] - r["noise_uc"])
    denoised = r["x"] + -sigmas[k] * noise_pred
    uncond_denoised = r["x"] + -sigmas[k] * r["noise_uc"]
    x1 = denoised + (r["x"] - uncond_denoised) / sigmas[k].item() * sigmas[k + 1]
    assert torch.equal(rec_split[k + 1]["x"], x1)
    # after k the history is the refiner's own: step k+1 sees step k's uncond denoised
    assert torch.equal(rec_split[k + 1]["old_denoised"], uncond_denoised)
    assert not torch.equal(split, full)


# ---- conditioning ---------------------------------------------------------------------------------------------------

class _Host:
    """What SDXL.refiner_conditions reads from a solver, without an engine."""
    def __init__(self):
        from cfgpp_b200 import config as C, latent_sdxl as L
        from cfgpp_b200.conditioning import SyntheticTextEncoder
        self.device, self.cfg = "cpu", C.sdxl_config()
        self.text_enc_2 = SyntheticTextEncoder(1280, 1280)
        self._L = L

    def _text_embed(self, *a, **k):
        return self._L.SDXL._text_embed(self, *a, **k)

    def _get_add_time_ids(self, *a, **k):
        return self._L.SDXL._get_add_time_ids(self, *a, **k)


@pytest.mark.parametrize("guidance,rows", [([0.6, 1.0], 4), (0.6, 4), (1.0, 2)])
def test_refiner_time_ids_and_rows(guidance, rows):
    from types import SimpleNamespace
    from cfgpp_b200 import config as C, latent_sdxl as L
    host = _Host()
    refiner = SimpleNamespace(cfg=C.sdxl_refiner_config(), text_enc=None)
    uc, c, add = L.SDXL.refiner_conditions(host, refiner, "", ["a cat", "a dog"], guidance, (1024, 1024), (0, 0),
                                           (1024, 1024), (0, 0), 6.0, 2.5, None, 2)
    assert uc.shape == c.shape == (2, 77, 1280)
    assert add["text_embeds"].shape == (rows, 1280) and add["time_ids"].shape == (rows, 5)
    pos, neg = [1024., 1024., 0., 0., 6.0], [1024., 1024., 0., 0., 2.5]
    t = add["time_ids"].float().tolist()
    if rows == 2:      # lambda in {0, 1}: the positive rows, broadcast over both halves
        assert t == [pos, pos]
    elif isinstance(guidance, list):  # per image: image 0 (0.6) takes the negative row, image 1 (1.0) the positive
        assert t == [neg, pos, pos, pos]
    else:
        assert t == [neg, neg, pos, pos]
    # the prompt pair went through the base's bigG tower: prompt1 only
    h, p = host.text_enc_2("a dog", "cpu")
    assert torch.equal(c[1:], h) and torch.equal(add["text_embeds"][-1:], p)
    # the base keeps its six ids
    base = L.SDXL._get_add_time_ids(host, (1024, 1024), (0, 0), (1024, 1024), torch.float16, 1280)
    assert base.tolist() == [[1024., 1024., 0., 0., 1024., 1024.]]


def test_refiner_rejected_by_other_solvers_before_any_work():
    from cfgpp_b200 import latent_sdxl as L
    assert set(L.REFINER_SOLVERS) <= set(L.__SOLVER__)
    for name, cls in L.__SOLVER__.items():
        fake = type(cls.__name__, (), {"supports_refiner": cls.supports_refiner, "schedule_kind": cls.schedule_kind})()
        if name in L.REFINER_SOLVERS:
            L.SDXL._check_refiner(fake)
        else:
            with pytest.raises(ValueError, match="ddim_cfg\\+\\+"):
                L.SDXL._check_refiner(fake)


# ---- checkpoints ----------------------------------------------------------------------------------------------------

def test_refiner_pipeline_directory(tmp_path, monkeypatch):
    from cfgpp_b200 import checkpoints as CK, text_encoder as TE
    for sub, name in (("unet", "diffusion_pytorch_model.fp16.safetensors"), ("vae", "diffusion_pytorch_model.safetensors"),
                      ("text_encoder_2", "model.fp16.safetensors")):
        (tmp_path / sub).mkdir()
        (tmp_path / sub / name).write_bytes(b"")
    with pytest.raises(FileNotFoundError) as e:
        CK.find_pipeline_files(tmp_path, "sdxl_refiner")
    assert "tokenizer_2" in str(e.value) and "text_encoder/" not in str(e.value) and "tokenizer/" not in str(e.value)
    (tmp_path / "tokenizer_2").mkdir()
    for name in ("vocab.json", "merges.txt"):
        (tmp_path / "tokenizer_2" / name).write_text("{}")
    f = CK.find_pipeline_files(tmp_path, "sdxl_refiner")
    assert set(f) == {"unet", "vae", "text_encoder_2", "tokenizer_2/vocab.json", "tokenizer_2/merges.txt"}
    # the base layout still needs text_encoder/ and tokenizer/
    with pytest.raises(FileNotFoundError, match="text_encoder/model"):
        CK.find_pipeline_files(tmp_path, "sdxl")
    calls = []
    monkeypatch.setattr(TE, "get_conditioner", lambda kind, *a, **k: calls.append((kind, a)) or kind)
    kw = CK.refiner_components(tmp_path, "cpu")
    assert kw["model_key"].endswith("unet/diffusion_pytorch_model.fp16.safetensors") and kw["text_encoder"] == "clip_bigg"
    assert calls[0][1][2].endswith("text_encoder_2/model.fp16.safetensors")
    (tmp_path / "unet" / "diffusion_pytorch_model.fp16.safetensors").unlink()
    with pytest.raises(FileNotFoundError, match="unet/diffusion_pytorch_model"):
        CK.refiner_components(tmp_path, "cpu")


def test_example_flags():
    """--denoising_end is an SDXL flag; the defaults leave the base-only path as it was."""
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    out = subprocess.run([sys.executable, "-m", "examples.text_to_img", "--model", "sd15", "--denoising_end", "0.8"],
                         cwd=root, capture_output=True, text=True, timeout=300)
    assert out.returncode != 0 and "--denoising_end needs --model sdxl" in out.stderr
