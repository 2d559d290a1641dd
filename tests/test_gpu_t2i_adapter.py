"""T2I-Adapter on the native backend: its kernels pinned on their own (pixel unshuffle, the 2x2 average pool, ReLU, the
gated add of the step graph), the adapter network against the oracle (tests/t2i_adapter_oracle.py) at the production
sizes, the UNet forward with features against the oracle UNet with `down_intrablock_additional_residuals`, and the plan's
behaviour around it (scale 0, factor 0 and detach, launches, per-entry words in fused trajectories, batching, a
ControlNet attached too, the solvers).

Tolerance of the forward comparisons: test_gpu_controlnet.py's (rel-L2 <= 5e-3 against the fp16-autocast oracle, and at
most 1.5x that oracle's own error against the fp32 oracle)."""
from ctypes import c_float, c_int, c_size_t

import pytest
import torch
import torch.nn.functional as F

import controlnet_oracle as CO
import production as P
import t2i_adapter_oracle as TO
from helpers import rel_l2

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
TOL = 5e-3


def _lib():
    from cfgpp_b200 import _native as nv
    return nv, nv.load()


# ---------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------
def _unshuffle_cases():
    """(factor, channels, H, W) of every T2I production size, once each (SD v1.5 and SD 2-base share 512²)."""
    from cfgpp_b200 import config as C, t2i_adapter as T
    out = []
    for name, h, w in P.t2i_sizes():
        f = T.t2i_adapter_config(C.CONFIGS[name]()).downscale_factor
        for c in (1, 3):
            if (f, c, 8 * h, 8 * w) not in out:
                out.append((f, c, 8 * h, 8 * w))
    return out


@pytest.mark.parametrize("f,C,H,W", _unshuffle_cases())
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_pixel_unshuffle_bit_exact(f, C, H, W, dtype):
    nv, lib = _lib()
    x = torch.rand(2, C, H, W, generator=torch.Generator().manual_seed(H + C)).to(dev, dtype)
    out = torch.empty(2, H // f, W // f, C * f * f, dtype=torch.float16, device=dev)
    nv.check(lib.cfgpp_op_pixel_unshuffle(nv.ptr(x), c_int(nv.dtype_code(x)), nv.ptr(out), c_int(2), c_int(C),
                                          c_int(H), c_int(W), c_int(f), nv.stream_ptr()))
    ref = F.pixel_unshuffle(x.half(), f).permute(0, 2, 3, 1)
    assert torch.equal(out, ref)


def _pool(x):
    nv, lib = _lib()
    B, H, W, C = x.shape
    out = torch.empty(B, H // 2, W // 2, C, dtype=torch.float16, device=dev)
    nv.check(lib.cfgpp_op_avgpool2x2(nv.ptr(x), nv.ptr(out), c_int(B), c_int(H), c_int(W), c_int(C), nv.stream_ptr()))
    return out


@pytest.mark.parametrize("B,H,W,C", [(1, 64, 64, 320), (8, 32, 48, 640), (2, 76, 52, 320), (1, 38, 26, 1280),
                                     (8, 16, 24, 1280), (1, 2, 2, 64)])
def test_avgpool2x2(B, H, W, C):
    """Bit for bit the fp16-rounded fp64 mean on integer-valued inputs (the fp32 sums are exact), within one fp16 ulp of
    it on random ones, and bit for bit torch's fp16 AvgPool2d(2, 2, ceil_mode=True) (the layer diffusers runs)."""
    g = torch.Generator().manual_seed(B * H + C)
    xi = torch.randint(-512, 512, (B, H, W, C), generator=g).half().to(dev)
    ref = F.avg_pool2d(xi.permute(0, 3, 1, 2).double(), 2).half().permute(0, 2, 3, 1)
    assert torch.equal(_pool(xi), ref)
    xr = torch.randn(B, H, W, C, generator=g).half().to(dev)
    got = _pool(xr)
    ref64 = F.avg_pool2d(xr.permute(0, 3, 1, 2).double(), 2).permute(0, 2, 3, 1)
    ulp = torch.abs(ref64.half().float()).clamp(min=2.0 ** -14) * 2.0 ** -10
    assert ((got.double() - ref64).abs() <= ulp.double()).all()
    pool = torch.nn.AvgPool2d(2, 2, ceil_mode=True)
    assert torch.equal(got, pool(xr.permute(0, 3, 1, 2)).permute(0, 2, 3, 1))


def test_relu_and_scale_bit_exact():
    nv, lib = _lib()
    g = torch.Generator().manual_seed(3)
    x = torch.cat([torch.randn(100003, generator=g) * 8, torch.zeros(5),
                   torch.tensor([65504., -65504., 6e-8, -6e-8, float("inf"), float("-inf")])]).half().to(dev)
    y = x.clone()
    nv.check(lib.cfgpp_op_relu(nv.ptr(y), c_size_t(y.numel()), nv.stream_ptr()))
    assert torch.equal(y, torch.relu(x))
    for s in (0.0, 0.37, 1.0, 2.5):
        out = torch.empty_like(x)
        nv.check(lib.cfgpp_op_scale(nv.ptr(x), c_float(s), nv.ptr(out), c_size_t(x.numel()), nv.stream_ptr()))
        ref = x * s
        ok = ~ref.isnan()  # inf * 0: NaN on both sides
        assert torch.equal(out.view(torch.int16)[ok], ref.view(torch.int16)[ok]) and torch.equal(out.isnan(), ~ok)


def _gated_add_cases():
    """(B, HW, C) of every tensor a feature lands on (`unet_placements`) at every T2I production size, for B images
    (UNet batch NB = 2B), once each."""
    from cfgpp_b200 import config as C, t2i_adapter as T
    out = []
    for name, h, w in P.t2i_sizes():
        for c, hh, ww in T.unet_placements(C.CONFIGS[name](), h, w):
            for B in P.T2I_ADAPTER_BATCHES:
                if (B, hh * ww, c) not in out:
                    out.append((B, hh * ww, c))
    return out


@pytest.mark.parametrize("B,HW,C", _gated_add_cases())
def test_gated_add(B, HW, C):
    """At every placement of the production sizes. On: bit for bit torch's fp16 add, rows b and B + b reading feature
    b. Off: not one bit written (-0.0 and NaN included)."""
    nv, lib = _lib()
    g = torch.Generator().manual_seed(B + C)
    h = torch.randn(2 * B, HW, C, generator=g).half().to(dev)
    h[0, 0, :4] = torch.tensor([-0.0, float("nan"), 65504., -0.0])
    feat = (torch.randn(B, HW, C, generator=g) * 3).half().to(dev)
    per = HW * C
    for on in (0, 1):
        word = torch.tensor([on], dtype=torch.int32, device=dev)
        out = h.clone()
        nv.check(lib.cfgpp_op_t2i_add(nv.ptr(out), nv.ptr(feat), c_int(2 * B), c_int(B), c_size_t(per), nv.ptr(word),
                                      nv.stream_ptr()))
        if on:
            ref = h + torch.cat([feat, feat])
            assert torch.equal(out.view(torch.int16)[~ref.isnan()], ref.view(torch.int16)[~ref.isnan()])
            assert out.isnan().equal(ref.isnan())
        else:
            assert torch.equal(out.view(torch.int16), h.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------
# the adapter network
# ---------------------------------------------------------------------------------------------------------------
def _adapter(name, in_channels=3, seed=7):
    from cfgpp_b200 import config as C, t2i_adapter as T
    ucfg = C.CONFIGS[name]()
    cfg = T.t2i_adapter_config(ucfg, in_channels)
    sd = T.synthetic_t2i_adapter_state_dict(cfg, seed=seed, device=dev)
    return ucfg, cfg, sd


def _adapter_cases():
    return [(name, h, w, b, c) for name, h, w in P.t2i_sizes() for b in P.T2I_ADAPTER_BATCHES
            for c in P.T2I_IN_CHANNELS]


@pytest.mark.parametrize("name,h,w,B,C", _adapter_cases())
def test_adapter_forward(name, h, w, B, C):
    from cfgpp_b200 import t2i_adapter as T
    _, cfg, sd = _adapter(name, C)
    ad = T.NativeT2IAdapter(cfg, sd, dev)
    image = torch.rand(B, C, 8 * h, 8 * w, generator=torch.Generator().manual_seed(B + h)).to(dev)
    got = [f.permute(0, 3, 1, 2).float() for f in ad.features(image, 0.8)]
    ad.close()
    m16 = TO.build_t2i_adapter(cfg, sd, torch.float16, dev)
    m32 = TO.build_t2i_adapter(cfg, sd, torch.float32, dev)
    with torch.no_grad():
        r16 = [f * 0.8 for f in m16(image.half())]
        r32 = [f * 0.8 for f in m32(image)]
    for k, (a, b16, b32) in enumerate(zip(got, r16, r32)):
        e16, e_ref = rel_l2(a, b16.float()), rel_l2(b16.float(), b32)
        print(f"{name} {8 * w}x{8 * h} B={B} C={C} feature {k}: rel-L2 vs fp16 {e16:.3e}, fp16 oracle vs fp32 "
              f"{e_ref:.3e}")
        assert tuple(a.shape) == tuple(b32.shape)
        assert e16 <= TOL and rel_l2(a, b32) <= 1.5 * e_ref + 1e-4


# ---------------------------------------------------------------------------------------------------------------
# the UNet with features
# ---------------------------------------------------------------------------------------------------------------
def _build(name, seed=1234):
    from cfgpp_b200 import config as C, t2i_adapter as T, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg = C.CONFIGS[name]()
    sd = Wt.synthetic_state_dict(cfg, seed=seed, device=dev)
    acfg = T.t2i_adapter_config(cfg)
    asd = T.synthetic_t2i_adapter_state_dict(acfg, seed=77, device=dev)
    return cfg, sd, NativeUNet(cfg, sd, dev), acfg, asd, T.NativeT2IAdapter(acfg, asd, dev)


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


def _oracle(cfg, sd, z, t, uc, c, add, feats16, feats32, cn=None):
    """(fp16-autocast, fp32) oracle outputs with the features (and optionally a ControlNet (cn_cfg, cn_sd, image, s))."""
    from oracle import unet as O
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
    out = []
    for dtype, feats in ((torch.float16, feats16), (torch.float32, feats32)):
        um = O.build_unet(CO.oracle_cfg(cfg), sd, dtype=dtype, device=dev)
        a = add if dtype == torch.float16 or add is None else {k: v.float() for k, v in add.items()}
        cx = ctx if dtype == torch.float16 else ctx.float()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=dtype == torch.float16):
            dres = mres = None
            if cn is not None:
                cm = CO.build_controlnet(cn[0], cn[1], dtype=dtype, device=dev)
                dres, mres = cm(z_in, t_in, cx, torch.cat([cn[2]] * 2), cn[3], a)
            r = TO.unet_forward(um, z_in, t_in, cx, a, feats, dres, mres)["sample"].float()
        out.append(r)
        del um
    return out


def forward_case(name, B, h, w, t, scale=0.8):
    cfg, sd, net, acfg, asd, ad = _build(name)
    z, uc, c, add, image = _inputs(cfg, B, h, w)
    feats = ad.features(image, scale)
    net.attach_t2i(len(feats))
    _bind(net, B, h, w, uc, c, add)
    net.set_t2i_features(feats)
    got = _native(net, z, t)
    net.attach_t2i(0)
    _bind(net, B, h, w, uc, c, add)
    plain = _native(net, z, t)
    net.close()
    ad.close()
    # the oracle UNets take the native adapter's features (the network is pinned on its own above), NCHW per CFG half
    f16 = [torch.cat([f.permute(0, 3, 1, 2)] * 2) for f in feats]
    r16, r32 = _oracle(cfg, sd, z, t, uc, c, add, f16, [f.float() for f in f16])
    e16, e_ref, e_plain = rel_l2(got, r16), rel_l2(r16, r32), rel_l2(plain, got)
    print(f"{name} {B}x{h}x{w}: rel-L2 vs fp16 oracle {e16:.3e}, vs fp32 {rel_l2(got, r32):.3e} (fp16 oracle vs fp32 "
          f"{e_ref:.3e}); with vs without the features {e_plain:.3e}")
    assert torch.isfinite(got).all()
    assert e16 <= TOL and rel_l2(got, r32) <= 1.5 * e_ref + 1e-4
    assert e_plain >= 10 * TOL  # the features matter: a skipped add cannot pass


@pytest.mark.parametrize("name,B,h,w,t", [("tiny_sd15", 1, 32, 32, 401), ("tiny_sd2", 2, 16, 16, 801),
                                          ("tiny_sdxl", 1, 32, 32, 601), ("tiny_sd15", 1, 16, 32, 301),
                                          ("tiny_sdxl", 2, 32, 16, 501)])
def test_t2i_forward_tiny(name, B, h, w, t):
    forward_case(name, B, h, w, t)


def test_t2i_forward_sd15_full_size():
    forward_case("sd15", 1, 64, 64, 501)


def test_t2i_forward_sdxl_full_size():
    forward_case("sdxl", 1, 128, 128, 501)


def test_scale_zero_factor_zero_and_detach_give_the_plain_unet_bit_for_bit():
    from cfgpp_b200 import schedule as S, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg, _, net, _, _, ad = _build("tiny_sdxl")
    z, uc, c, add, image = _inputs(cfg, 1, 32, 32)
    fresh = NativeUNet(cfg, Wt.synthetic_state_dict(cfg, seed=1234, device=dev), dev)
    _bind(fresh, 1, 32, 32, uc, c, add)
    never = _native(fresh, z, 500)
    steps = S.ddim_cfgpp_steps(S.Schedule.make(4), 0.6, sdxl_indexing=True)
    _, never_traj = fresh.run_trajectory(S.STEP_DDIM_CFGPP, torch.float32, steps, z)
    net.attach_t2i(4)
    _bind(net, 1, 32, 32, uc, c, add)
    net.set_t2i_features(ad.features(image, 0.0))
    assert torch.equal(_native(net, z, 500), never)  # scale 0
    assert net.launches_per_step == fresh.launches_per_step + 4
    net.set_t2i_features(ad.features(image, 1.0))
    assert not torch.equal(_native(net, z, 500), never)
    net.set_t2i_active(False)  # factor 0: the word is off
    assert torch.equal(_native(net, z, 500), never)
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
    net.set_t2i_steps([False] * len(steps))
    net.set_state(z)
    net.run_steps()
    assert torch.equal(net.get_state(0), never_traj)
    net.set_t2i_active(True)
    net.attach_t2i(0)
    _bind(net, 1, 32, 32, uc, c, add)
    assert torch.equal(_native(net, z, 500), never)
    assert net.plan_stats == fresh.plan_stats and net.launches_per_step == fresh.launches_per_step
    fresh.close()
    net.close()
    ad.close()


def test_run_without_features_fails_and_counts_are_refused():
    from cfgpp_b200 import _native as nv
    cfg, _, net, _, _, ad = _build("tiny_sd15")
    z, uc, c, add, image = _inputs(cfg, 1, 16, 16)
    with pytest.raises(nv.NativeError, match="num_levels"):
        net.attach_t2i(3)
    net.attach_t2i(4)
    _bind(net, 1, 16, 16, uc, c, add)
    with pytest.raises(nv.NativeError, match="set_t2i_features"):
        net.predict_noise(z, 500.0)
    net.set_t2i_features(ad.features(image))
    net.predict_noise(z, 500.0)
    net.close()
    ad.close()


@pytest.mark.parametrize("kind", ["ddim_cfg++", "dpm++_2s_a"])
def test_fused_trajectory_with_factor_cut_equals_callback_path(kind):
    """A factor of 0.5: the fused graph (one word per entry, both entries of a 2S step sharing theirs) equals the
    un-fused entry-by-entry path bit for bit, and differs from the trajectory with the features on throughout."""
    from cfgpp_b200 import kdiffusion as K, schedule as S, t2i_adapter as T
    cfg, _, net, _, _, ad = _build("tiny_sd15")
    z, uc, c, add, image = _inputs(cfg, 1, 32, 32)
    net.attach_t2i(4)
    _bind(net, 1, 32, 32, uc, c, add)
    net.set_t2i_features(ad.features(image))
    noise = None
    if kind == "ddim_cfg++":
        mode, dtype, x = S.STEP_DDIM_CFGPP, torch.float32, z
        steps = S.ddim_cfgpp_steps(S.Schedule.make(10), 0.6, sdxl_indexing=False)
    else:
        mode, dtype = S.STEP_DPMPP2M_CFGPP, torch.float16
        sigmas = K.get_sigmas_karras(8, 0.03, 14.6, rho=7.)
        steps, slots = S.kd_ancestral_steps(sigmas, lambda s: torch.clamp(s * 60, max=999.0), 0.6, True, two_s=True)
        noise = torch.randn(slots, 1, 4, 32, 32, generator=torch.Generator().manual_seed(2)).half().to(dev)
        x = (z * sigmas[0]).half()
        assert any(st.coef.second_order & S.KD_2S_FINAL for st in steps)
    flags = T.entry_flags(steps, 0.5)
    assert True in flags and False in flags

    def fused(fl):
        net.set_schedule(mode, dtype, steps)
        net.set_t2i_steps(fl)
        if noise is not None:
            net.set_noise(noise)
        net.set_state(x)
        net.run_steps()
        return net.get_state(0)

    cut = fused(flags)
    net.set_schedule(mode, dtype, steps)
    if noise is not None:
        net.set_noise(noise)
    net.set_state(x)
    for i, st in enumerate(steps):
        net.set_t2i_active(flags[i])
        _, zt = net.callback_step(i, st)
    assert torch.equal(zt, cut)
    assert not torch.equal(fused([True] * len(steps)), cut)
    net.close()
    ad.close()


def test_batched_adapter_images_rows_independent():
    """Image b's features reach prompt b only, in both CFG halves."""
    cfg, _, net, _, _, ad = _build("tiny_sd15")
    z, uc, c, add, image = _inputs(cfg, 4, 16, 16)
    net.attach_t2i(4)
    _bind(net, 4, 16, 16, uc, c, add)
    net.set_t2i_features(ad.features(image))
    eu, ec = net.predict_noise(z, 700.0)
    for i in (0, 3):
        net.prepare(1, 16, 16)
        net.set_prompt(torch.cat([uc[i:i + 1], c[i:i + 1]]))
        net.set_t2i_features(ad.features(image[i:i + 1].contiguous()))
        su, sc = net.predict_noise(z[i:i + 1], 700.0)
        assert rel_l2(su, eu[i:i + 1]) < 1e-3 and rel_l2(sc, ec[i:i + 1]) < 1e-3
    net.close()
    ad.close()


def test_with_a_controlnet_attached():
    """A T2I-Adapter and a ControlNet together against the oracle with both, the adapter's adds first."""
    from cfgpp_b200 import controlnet as CN
    cfg, sd, net, _, _, ad = _build("tiny_sdxl")
    cn_cfg = CN.controlnet_config(cfg)
    cn_sd = CN.synthetic_controlnet_state_dict(cn_cfg, seed=99, device=dev)
    cn = CN.NativeControlNet(cn_cfg, cn_sd, dev)
    z, uc, c, add, image = _inputs(cfg, 1, 32, 32)
    feats = ad.features(image, 0.9)
    net.attach_controlnet(cn)
    net.attach_t2i(4)
    _bind(net, 1, 32, 32, uc, c, add)
    net.set_control_image(image)
    net.set_control_scale(0.7)
    net.set_t2i_features(feats)
    got = _native(net, z, 450)
    net.close()
    cn.close()
    ad.close()
    f16 = [torch.cat([f.permute(0, 3, 1, 2)] * 2) for f in feats]
    r16, r32 = _oracle(cfg, sd, z, 450, uc, c, add, f16, [f.float() for f in f16], (cn_cfg, cn_sd, image, 0.7))
    e16, e_ref = rel_l2(got, r16), rel_l2(r16, r32)
    print(f"T2I + ControlNet: rel-L2 vs fp16 oracle {e16:.3e}, fp16 oracle vs fp32 {e_ref:.3e}")
    assert e16 <= TOL and rel_l2(got, r32) <= 1.5 * e_ref + 1e-4


class _LatentVAE:
    def __init__(self):
        self.latents = []

    def decode(self, z):
        self.latents.append(z.detach().clone())
        return torch.zeros(z.shape[0], 3, 8 * z.shape[2], 8 * z.shape[3], device=z.device)


@pytest.mark.parametrize("family,method", [("sd", "ddim_cfg++"), ("sd", "dpm++_2s_a_cfg++"), ("sd", "dpm++_2m"),
                                           ("sdxl", "ddim"), ("sdxl", "dpm++_2m_cfgpp"), ("sdxl", "euler_cfg++")])
def test_solver_sample_with_t2i_adapter(family, method):
    """sample(t2i_adapter=...) with a factor cut: the fused trajectory and the callback path agree; the adapter moves
    the image; a later call without it on the shared engine is the plain image again, bit for bit."""
    from types import SimpleNamespace
    from cfgpp_b200 import config as C, latent_diffusion as LD, latent_sdxl as LX, t2i_adapter as T, weights as Wt
    cfg = C.tiny_sd15_config() if family == "sd" else C.tiny_sdxl_config()
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    vae = _LatentVAE()
    s = (LD if family == "sd" else LX).get_solver(method, solver_config=SimpleNamespace(num_sampling=6), device=dev,
                                                   unet_config=cfg, state_dict=sd, vae=vae)
    hw = cfg.sample_size
    g = torch.Generator().manual_seed(4)
    zT = torch.randn(2, 4, hw, hw, generator=g)
    image = torch.rand(2, 1, 8 * hw, 8 * hw, generator=g)
    ad = T.T2IAdapter("synthetic-sketch", dev, base_cfg=cfg, in_channels=1)
    kw = dict(t2i_adapter=ad, t2i_adapter_image=image, adapter_conditioning_scale=0.9,
              adapter_conditioning_factor=0.5)

    def run(**kw):
        torch.manual_seed(9)  # the ancestral noise
        if family == "sd":
            s.sample(cfg_guidance=0.6, prompt=["", ["a cat", "a dog"]], zT=zT, **kw)
        else:
            s.sample(prompt1=["", ["a cat", "a dog"]], prompt2=["", ["a cat", "a dog"]], cfg_guidance=0.6,
                     target_size=(8 * hw, 8 * hw), zT=zT, **kw)
        return vae.latents[-1].float()

    plain = run()
    fused = run(**kw)
    callback = run(callback_fn=lambda i, t, k: k, **kw)
    again = run()
    e_cb, moved = rel_l2(callback, fused), rel_l2(fused, plain)
    print(f"{family} {method}: callback vs fused rel-L2 {e_cb:.3e}, with vs without the T2I-Adapter {moved:.3e}")
    assert torch.isfinite(fused).all() and moved >= 10 * TOL
    if "ddim" in method:  # both paths run the step kernel
        assert torch.equal(callback, fused)
    else:  # the callback path is the op-by-op torch loop
        assert e_cb <= 1e-2
    assert torch.equal(again, plain)
    with pytest.raises(ValueError, match="channels"):
        run(t2i_adapter=ad, t2i_adapter_image=torch.rand(1, 3, 8 * hw, 8 * hw))
    ad.engine.close()
