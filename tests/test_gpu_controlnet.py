"""ControlNet on the native backend: each new piece pinned on its own (the scaled-residual GEMM epilogue, conv_in with an
addend, the conditioning embedding), then the whole attached forward against the oracle ControlNet + oracle UNet with
residuals (tests/controlnet_oracle.py) on the same seeded weights, and the plan's behaviour around it (scale zero,
detach, per-entry scale tables in fused trajectories, batching).

Tolerance of the forward comparisons: test_gpu_unet.py's (rel-L2 <= 5e-3 against the fp16-autocast oracle, and at most
1.5x that oracle's own error against the fp32 oracle)."""
import pytest
import torch

import controlnet_oracle as CO
from helpers import rel_l2

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
TOL = 5e-3


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g).half().to(dev)


# ---------------------------------------------------------------------------------------------------------------
# scaled-residual epilogue
# ---------------------------------------------------------------------------------------------------------------
def _scaled_reference(a, w, bias, addend, s):
    acc = (a.double() @ w.double().T).float()  # integer-valued: exact in fp32
    t = (acc + bias.float()).half()
    ts = (t.float() * torch.tensor(s, dtype=torch.float32)).half()
    return (addend.float() + ts.float()).half()


@pytest.mark.parametrize("s", [0.0, 0.5, 0.37, 1.0, 2.0])
@pytest.mark.parametrize("M,C", [(2 * 1 * 64 * 64, 320), (2 * 2 * 32 * 32, 640), (2 * 1 * 16 * 16, 1280),
                                 (2 * 4 * 8 * 8, 1280), (300, 128)])
def test_scaled_residual_epilogue_bit_exact(M, C, s):
    """Zero-conv shapes (C = 320 / 640 / 1280 at their latent sizes, M = 2 B HW) and a ragged M: bit-exact against
    fp16(addend + fp16(fp16(acc + bias) * s)), in place and out of place."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(C + M)
    a, w = _ints((M, C), -2, 2, g), _ints((C, C), -1, 1, g)
    bias, addend = _ints((C,), -8, 8, g) * 0.5, _ints((M, C), -64, 64, g) * 0.25
    scale = torch.tensor([s], dtype=torch.float32, device=dev)
    ref = _scaled_reference(a.cpu(), w.cpu(), bias.cpu(), addend.cpu(), s).to(dev)
    out = nv.op_linear_scaled_residual(a, w, addend, scale, bias)
    assert torch.equal(out, ref)
    inplace = addend.clone()
    nv.op_linear_scaled_residual(a, w, inplace, scale, bias, out=inplace)
    assert torch.equal(inplace, ref)
    if s == 1.0:  # the unscaled addend epilogue of today, bit for bit
        assert torch.equal(out, nv.op_linear(a, w, bias, addend))
        assert torch.equal(nv.op_linear_scaled_residual(a, w, addend, None, bias), out)
    if s == 0.0:
        assert torch.equal(out, addend)


# ---------------------------------------------------------------------------------------------------------------
# conv_in + addend
# ---------------------------------------------------------------------------------------------------------------
def _conv_in_cases():
    """The earlier shapes, then every latent size of `production.CONTROLNET_SIZES` at C0 = 320 for 2 images."""
    import production as P
    cases = [(1, 64, 64, 320), (2, 16, 24, 64)]
    for _, h, w in P.controlnet_sizes():
        if (2, h, w, 320) not in cases:
            cases.append((2, h, w, 320))
    return cases


@pytest.mark.parametrize("B,H,W,C", _conv_in_cases())
def test_conv_in_with_addend(B, H, W, C):
    """fp16(fp16(conv_in(z)) + addend) on every repetition, per element against fp64: the fp32 sum of 36 products and
    the bias (37 roundings in a fixed order, E_acc = 38·u·(Σ|w·x| + |b|)), ½ ulp for the conv's fp16 rounding, then
    the add (u·|ref| and its ½ ulp); and bit for bit against conv_in followed by the fp16 add."""
    from cfgpp_b200 import _native as nv
    from test_gpu_norms import Gate, ulp16
    u = 2.0 ** -24
    g = torch.Generator().manual_seed(11 + B * H + W)
    z = torch.randn(B, 4, H, W, generator=g).to(dev)
    w = (torch.randn(C, 4, 3, 3, generator=g) * 0.3).half().to(dev)
    bias = (torch.randn(C, generator=g) * 0.1).half().to(dev)
    addend = torch.randn(B, H, W, C, generator=g).half().to(dev)
    got = nv.op_conv_in_add(z, w.reshape(C, 36), bias, addend, reps=2)
    plain = nv.op_conv_in(z, w.reshape(C, 36), bias, reps=2)
    want = (plain.float() + torch.cat([addend] * 2).float()).half()
    assert torch.equal(got, want)
    assert torch.equal(got[:B], got[B:]), "the two repetitions differ"
    zh = z.half().double()
    conv64 = torch.nn.functional.conv2d(zh, w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    mag = torch.nn.functional.conv2d(zh.abs(), w.double().abs(), bias.double().abs(), padding=1).permute(0, 2, 3, 1)
    e_t = 38 * u * mag
    e_t = e_t + 0.5 * ulp16(conv64.abs() + e_t)
    ref = conv64 + addend.double()
    gate = Gate(f"conv_in+addend {B}x{H}x{W} C{C}")
    gate.add(got[:B].double(), ref, e_t + u * ref.abs())
    gate.done("controlnet")


# ---------------------------------------------------------------------------------------------------------------
# the attached forward
# ---------------------------------------------------------------------------------------------------------------
def _build(name, seed=1234, cn_seed=99):
    from cfgpp_b200 import config as C, controlnet as CN, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg = C.CONFIGS[name]()
    sd = Wt.synthetic_state_dict(cfg, seed=seed, device=dev)
    cn_cfg = CN.controlnet_config(cfg)
    cn_sd = CN.synthetic_controlnet_state_dict(cn_cfg, seed=cn_seed, device=dev)
    return cfg, sd, NativeUNet(cfg, sd, dev), cn_cfg, cn_sd, CN.NativeControlNet(cn_cfg, cn_sd, dev)


def _inputs(cfg, B, h, w, seed=5, dup=True):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 4, h, w, generator=g).to(dev)
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    add = None
    if cfg.addition_embed_type == "text_time":
        rows = 2 * B if dup else B
        add = {"text_embeds": torch.randn(rows, cfg.pooled_dim, generator=g).half().to(dev),
               "time_ids": torch.tensor([[8. * h, 8. * w, 0, 0, 8. * h, 8. * w]] * rows).half().to(dev)}
    image = torch.rand(B, 3, 8 * h, 8 * w, generator=g).to(dev)
    return z, uc, c, add, image


def _bind(net, B, h, w, uc, c, add):
    net.prepare(B, h, w)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"] if add else None, add["time_ids"].float() if add else None)


def _native(net, z, t):
    eu, ec = net.predict_noise(z, float(t))
    return torch.cat([eu, ec]).float()


def forward_case(name, B, h, w, t, dup=True, scale=0.8):
    from oracle import unet as O
    cfg, sd, net, cn_cfg, cn_sd, cn = _build(name)
    z, uc, c, add, image = _inputs(cfg, B, h, w, dup=dup)
    net.attach_controlnet(cn)
    _bind(net, B, h, w, uc, c, add)
    net.set_control_image(image)
    net.set_control_scale(scale)
    got = _native(net, z, t)
    net.attach_controlnet(None)
    _bind(net, B, h, w, uc, c, add)
    plain = _native(net, z, t)
    net.close()
    cn.close()
    z_in, t_in, ctx, img2 = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c]), torch.cat([image] * 2)
    um = O.build_unet(CO.oracle_cfg(cfg), sd, dtype=torch.float16, device=dev)
    cm = CO.build_controlnet(cn_cfg, cn_sd, dtype=torch.float16, device=dev)
    with torch.autocast("cuda", dtype=torch.float16), torch.no_grad():
        dres, mres = cm(z_in, t_in, ctx, img2, scale, add)
        r16 = CO.unet_forward(um, z_in, t_in, ctx, add, dres, mres)["sample"].float()
    del um, cm
    um = O.build_unet(CO.oracle_cfg(cfg), sd, dtype=torch.float32, device=dev)
    cm = CO.build_controlnet(cn_cfg, cn_sd, dtype=torch.float32, device=dev)
    add32 = {k: v.float() for k, v in add.items()} if add else None
    with torch.no_grad():
        dres, mres = cm(z_in, t_in, ctx.float(), img2, scale, add32)
        r32 = CO.unet_forward(um, z_in, t_in, ctx.float(), add32, dres, mres)["sample"]
    del um, cm
    e16, e_ref, e_plain = rel_l2(got, r16), rel_l2(r16, r32), rel_l2(plain, got)
    print(f"{name} {B}x{h}x{w}: rel-L2 vs fp16 oracle {e16:.3e}, vs fp32 {rel_l2(got, r32):.3e} "
          f"(fp16 oracle vs fp32 {e_ref:.3e}); with vs without the ControlNet {e_plain:.3e}")
    assert torch.isfinite(got).all()
    assert e16 <= TOL
    assert rel_l2(got, r32) <= 1.5 * e_ref + 1e-4
    assert e_plain >= 10 * TOL  # the residuals matter: a skipped add cannot pass


@pytest.mark.parametrize("name,B,h,w,t,dup", [("tiny_sd15", 1, 32, 32, 401, True), ("tiny_sd2", 2, 16, 16, 801, True),
                                              ("tiny_sdxl", 1, 32, 32, 601, True), ("tiny_sdxl", 1, 32, 32, 999, False),
                                              ("tiny_sd15", 1, 16, 32, 301, True)])
def test_controlnet_forward_tiny(name, B, h, w, t, dup):
    forward_case(name, B, h, w, t, dup)


def test_controlnet_forward_sd15_full_size():
    forward_case("sd15", 1, 64, 64, 501)


def test_controlnet_forward_sdxl_full_size():
    forward_case("sdxl", 1, 128, 128, 501)


@pytest.mark.parametrize("name,hw", [("sd15", 64), ("sdxl", 128)])
def test_conditioning_embedding(name, hw):
    """The once-per-image CNN at 512^2 / 1024^2 against the fp16-autocast and fp32 oracles."""
    from cfgpp_b200 import config as C, controlnet as CN
    cn_cfg = CN.controlnet_config(C.CONFIGS[name]())
    specs = [s for s in CN.controlnet_param_specs(cn_cfg) if s[0].startswith("controlnet_cond_embedding.")]
    from cfgpp_b200.weights import synthetic_from_specs
    emb_sd = synthetic_from_specs(specs, 3, dev)
    sd = CN.synthetic_controlnet_state_dict(cn_cfg, seed=3, device=dev)
    sd.update(emb_sd)
    cn = CN.NativeControlNet(cn_cfg, sd, dev)
    image = torch.rand(2, 3, 8 * hw, 8 * hw, generator=torch.Generator().manual_seed(1)).to(dev)
    got = cn.embed(image).permute(0, 3, 1, 2).float()
    cn.close()
    m = CO.ControlNetConditioningEmbedding(cn_cfg.unet.block_out_channels[0], cn_cfg.conditioning_embedding_out_channels)
    m.load_state_dict({k[len("controlnet_cond_embedding."):]: v.float() for k, v in emb_sd.items()})
    m = m.to(dev)
    with torch.no_grad():
        r32 = m(image)
        with torch.autocast("cuda", dtype=torch.float16):
            r16 = m(image).float()
    e16, e_ref = rel_l2(got, r16), rel_l2(r16, r32)
    print(f"{name} conditioning embedding: rel-L2 vs fp16 oracle {e16:.3e}, fp16 oracle vs fp32 {e_ref:.3e}")
    assert e16 <= TOL and rel_l2(got, r32) <= 1.5 * e_ref + 1e-4


# ---------------------------------------------------------------------------------------------------------------
# plan behaviour
# ---------------------------------------------------------------------------------------------------------------
def test_scale_zero_and_detach_give_the_plain_unet_bit_for_bit():
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg, sd, net, _, _, cn = _build("tiny_sdxl")
    z, uc, c, add, image = _inputs(cfg, 1, 32, 32)
    fresh = NativeUNet(cfg, Wt.synthetic_state_dict(cfg, seed=1234, device=dev), dev)
    _bind(fresh, 1, 32, 32, uc, c, add)
    never = _native(fresh, z, 500)
    net.attach_controlnet(cn)
    _bind(net, 1, 32, 32, uc, c, add)
    net.set_control_image(image)
    net.set_control_scale(0.0)
    assert torch.equal(_native(net, z, 500), never)
    net.set_control_scale(1.0)
    assert not torch.equal(_native(net, z, 500), never)
    stats_cn = net.plan_stats
    net.attach_controlnet(None)
    _bind(net, 1, 32, 32, uc, c, add)
    assert torch.equal(_native(net, z, 500), never)
    assert net.plan_stats == fresh.plan_stats and net.launches_per_step == fresh.launches_per_step
    assert stats_cn["step_flops"] > 1.2 * fresh.plan_stats["step_flops"]
    fresh.close()
    net.close()
    cn.close()


def test_run_without_control_image_fails():
    from cfgpp_b200 import _native as nv
    cfg, _, net, _, _, cn = _build("tiny_sd15")
    z, uc, c, add, image = _inputs(cfg, 1, 16, 16)
    net.attach_controlnet(cn)
    _bind(net, 1, 16, 16, uc, c, add)
    with pytest.raises(nv.NativeError, match="set_control_image"):
        net.predict_noise(z, 500.0)
    net.set_control_image(image)
    net.predict_noise(z, 500.0)
    net.close()
    cn.close()


def test_fused_trajectory_with_scale_table_equals_callback_path():
    """A DDIM trajectory with a control_guidance_start / end table: the fused graph equals the un-fused callback path
    bit for bit, and a new table between two runs takes effect without a re-prepare."""
    from cfgpp_b200 import controlnet as CN, schedule as S
    cfg, _, net, _, _, cn = _build("tiny_sd15")
    z, uc, c, add, image = _inputs(cfg, 1, 32, 32)
    net.attach_controlnet(cn)
    _bind(net, 1, 32, 32, uc, c, add)
    net.set_control_image(image)
    steps = S.ddim_cfgpp_steps(S.Schedule.make(10), 0.6, sdxl_indexing=False)
    table = CN.control_scales(len(steps), 0.9, 0.1, 0.7)
    assert table[0] == 0.0 and table[1] == 0.9 and table[-1] == 0.0
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
    net.set_control_scales(table)
    net.set_state(z)
    net.run_steps()
    fused = net.get_state(0)
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
    net.set_state(z)
    for i, st in enumerate(steps):
        net.set_control_scale(table[i])
        _, zt = net.callback_step(i, st)
    assert torch.equal(zt, fused)
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
    net.set_control_scales([0.0] * len(steps))
    net.set_state(z)
    net.run_steps()
    zero = net.get_state(0)
    net.attach_controlnet(None)
    _bind(net, 1, 32, 32, uc, c, add)
    _, plain = net.run_trajectory(S.STEP_DDIM_CFGPP, torch.float32, steps, z)
    assert torch.equal(zero, plain) and not torch.equal(zero, fused)
    net.close()
    cn.close()


def test_batched_control_images_rows_independent():
    cfg, _, net, _, _, cn = _build("tiny_sd15")
    z, uc, c, add, image = _inputs(cfg, 4, 16, 16)
    net.attach_controlnet(cn)
    _bind(net, 4, 16, 16, uc, c, add)
    net.set_control_image(image)
    eu, ec = net.predict_noise(z, 700.0)
    for i in (0, 3):
        net.prepare(1, 16, 16)
        net.set_prompt(torch.cat([uc[i:i + 1], c[i:i + 1]]))
        net.set_control_image(image[i:i + 1].contiguous())
        su, sc = net.predict_noise(z[i:i + 1], 700.0)
        assert rel_l2(su, eu[i:i + 1]) < 1e-3 and rel_l2(sc, ec[i:i + 1]) < 1e-3
    net.close()
    cn.close()


def test_attach_refuses_a_mismatched_controlnet():
    from cfgpp_b200 import _native as nv, config as C, controlnet as CN, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    sd15 = C.tiny_sd15_config()
    net = NativeUNet(sd15, Wt.synthetic_state_dict(sd15, device=dev), dev)
    xl_cfg = CN.controlnet_config(C.tiny_sdxl_config())
    cn = CN.NativeControlNet(xl_cfg, CN.synthetic_controlnet_state_dict(xl_cfg, device=dev), dev)
    with pytest.raises(nv.NativeError, match="num_levels"):
        net.attach_controlnet(cn)
    net.close()
    cn.close()


# ---------------------------------------------------------------------------------------------------------------
# VE-cast trajectories with a scale table, LoRA under an attached ControlNet, the solvers
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["dpm++_2m", "dpm++_2s_a"])
def test_kdiffusion_trajectory_with_scale_table_equals_callback_path(kind):
    """DPM++ 2M and ancestral DPM-Solver++(2S) (two schedule entries per step sharing their step's scale) with a start /
    end table: the fused graph equals the un-fused entry-by-entry path bit for bit."""
    from cfgpp_b200 import controlnet as CN, kdiffusion as K, schedule as S
    cfg, _, net, _, _, cn = _build("tiny_sd15")
    z, uc, c, add, image = _inputs(cfg, 1, 32, 32)
    net.attach_controlnet(cn)
    _bind(net, 1, 32, 32, uc, c, add)
    net.set_control_image(image)
    sigmas = K.get_sigmas_karras(8, 0.03, 14.6, rho=7.)
    ts = lambda s: torch.clamp(s * 60, max=999.0)  # noqa: E731
    noise = None
    if kind == "dpm++_2m":
        steps = S.kd_steps(sigmas, ts, 0.6, True, second_order=True, diff_guided=True)
    else:
        steps, slots = S.kd_ancestral_steps(sigmas, ts, 0.6, True, two_s=True)
        noise = torch.randn(slots, 1, 4, 32, 32, generator=torch.Generator().manual_seed(2)).half().to(dev)
        assert any(st.coef.second_order & S.KD_2S_FINAL for st in steps)
    table = CN.entry_scales(steps, 0.9, 0.2, 0.7)
    assert 0.0 in table and 0.9 in table
    x = (z * sigmas[0]).half()
    net.set_schedule(S.STEP_DPMPP2M_CFGPP, torch.float16, steps, control_scales=table)
    if noise is not None:
        net.set_noise(noise)
    net.set_state(x)
    net.run_steps()
    fused = net.get_state(0)
    net.set_schedule(S.STEP_DPMPP2M_CFGPP, torch.float16, steps)
    if noise is not None:
        net.set_noise(noise)
    net.set_state(x)
    for i, st in enumerate(steps):
        net.set_control_scale(table[i])
        _, zt = net.callback_step(i, st)
    assert torch.equal(zt, fused)
    net.close()
    cn.close()


def test_lora_merges_with_a_controlnet_attached():
    """A UNet LoRA loaded while a ControlNet is attached merges into the UNet only: the attached forward matches the
    oracle UNet with the merged weights plus the untouched oracle ControlNet; clearing it restores the output bit for
    bit."""
    from oracle import unet as O
    from cfgpp_b200 import _native as nv
    from test_gpu_lora import random_adapter
    cfg, sd, net, cn_cfg, cn_sd, cn = _build("tiny_sdxl")
    z, uc, c, add, image = _inputs(cfg, 1, 32, 32)
    net.attach_controlnet(cn)
    _bind(net, 1, 32, 32, uc, c, add)
    net.set_control_image(image)
    net.set_control_scale(0.8)
    before = _native(net, z, 500)
    adapter = random_adapter(cfg, 8, 3)
    net.add_lora(adapter, 0.7)
    with pytest.raises(nv.NativeError, match="set_prompt"):
        net.predict_noise(z, 500.0)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
    got = _native(net, z, 500)
    merged = dict(sd)
    for key, (down, up, alpha) in adapter.targets.items():
        w = sd[key]
        delta = (0.7 * alpha / down.shape[0]) * (up.float().to(dev) @ down.float().to(dev))
        merged[key] = (w.float() + delta.reshape(w.shape)).half()
    z_in, t_in, ctx, img2 = torch.cat([z] * 2), torch.tensor(500, device=dev), torch.cat([uc, c]), torch.cat([image] * 2)
    um = O.build_unet(CO.oracle_cfg(cfg), merged, dtype=torch.float16, device=dev)
    cm = CO.build_controlnet(cn_cfg, cn_sd, dtype=torch.float16, device=dev)
    with torch.autocast("cuda", dtype=torch.float16), torch.no_grad():
        dres, mres = cm(z_in, t_in, ctx, img2, 0.8, add)
        r16 = CO.unet_forward(um, z_in, t_in, ctx, add, dres, mres)["sample"].float()
    e, moved = rel_l2(got, r16), rel_l2(got, before)
    print(f"LoRA + ControlNet: rel-L2 vs fp16 oracle {e:.3e}, moved by the adapter {moved:.3e}")
    assert e <= TOL and moved >= 10 * TOL
    net.clear_lora()
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
    assert torch.equal(_native(net, z, 500), before)
    net.close()
    cn.close()


class _LatentVAE:
    def __init__(self):
        self.latents = []

    def decode(self, z):
        self.latents.append(z.detach().clone())
        return torch.zeros(z.shape[0], 3, 8 * z.shape[2], 8 * z.shape[3], device=z.device)


@pytest.mark.parametrize("family,method", [("sd", "ddim_cfg++"), ("sd", "dpm++_2s_a_cfg++"), ("sd", "dpm++_2m"),
                                           ("sdxl", "ddim"), ("sdxl", "dpm++_2m_cfgpp"), ("sdxl", "euler_cfg++")])
def test_solver_sample_with_controlnet(family, method):
    """sample(controlnet=...): the fused trajectory and the callback path give the same image; the ControlNet moves
    it; a later call without controlnet= on the shared engine is the uncontrolled image again, bit for bit."""
    from types import SimpleNamespace
    from cfgpp_b200 import config as C, controlnet as CN, latent_diffusion as LD, latent_sdxl as LX, weights as Wt
    cfg = C.tiny_sd15_config() if family == "sd" else C.tiny_sdxl_config()
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    vae = _LatentVAE()
    s = (LD if family == "sd" else LX).get_solver(method, solver_config=SimpleNamespace(num_sampling=6), device=dev,
                                                   unet_config=cfg, state_dict=sd, vae=vae)
    hw = cfg.sample_size
    g = torch.Generator().manual_seed(4)
    zT = torch.randn(2, 4, hw, hw, generator=g)
    image = torch.rand(1, 3, 8 * hw, 8 * hw, generator=g)
    cn = CN.ControlNet("synthetic-controlnet", dev, base_cfg=cfg)
    ctl = dict(controlnet=cn, control_image=image, controlnet_conditioning_scale=0.9, control_guidance_start=0.2,
               control_guidance_end=0.8)

    def run(**kw):
        torch.manual_seed(9)  # the ancestral noise
        if family == "sd":
            s.sample(cfg_guidance=0.6, prompt=["", ["a cat", "a dog"]], zT=zT, **kw)
        else:
            s.sample(prompt1=["", ["a cat", "a dog"]], prompt2=["", ["a cat", "a dog"]], cfg_guidance=0.6,
                     target_size=(8 * hw, 8 * hw), zT=zT, **kw)
        return vae.latents[-1].float()

    plain = run()
    fused = run(**ctl)
    callback = run(callback_fn=lambda i, t, kw: kw, **ctl)
    again = run()
    e_cb, moved = rel_l2(callback, fused), rel_l2(fused, plain)
    print(f"{family} {method}: callback vs fused rel-L2 {e_cb:.3e}, with vs without the ControlNet {moved:.3e}")
    assert torch.isfinite(fused).all() and moved >= 10 * TOL
    if "ddim" in method:  # both paths run the step kernel
        assert torch.equal(callback, fused)
    else:  # the callback path is the op-by-op torch loop
        assert e_cb <= 1e-2
    assert torch.equal(again, plain) and s.unet.controlnet is None
    with pytest.raises(ValueError, match="resized"):
        run(controlnet=cn, control_image=torch.rand(1, 3, 8 * hw, 4 * hw))
    cn.engine.close()
