"""IP-Adapter Plus on the GPU: the vision tower's hidden-state output, the Resampler's LayerNorm-concat kernel
(`ln_concat_kernel`, norm.cu), the Resampler's attention and LayerNorm launches at the production sizes under the
existing per-element gates (its GEMMs are in `test_gpu_gemm.py`'s production lists), and the Plus adapter inside the
UNet executor and through sample(). Every measured error is printed."""
import pytest
import torch

import ip_adapter_plus_oracle as PO
import production as P
from test_gpu_ip_adapter import TOL, _bind, _captures, _inputs, _native, _net, _trajectory, dev

pytestmark = pytest.mark.gpu


def _geometry(name):
    """(Resampler geometry, token width D, hidden-state rows T) of the Plus adapter of IP_PLUS_ADAPTERS for `name`."""
    from cfgpp_b200 import config as C, ip_adapter as IP
    cfg, E = C.CONFIGS[name](), dict(P.IP_PLUS_ADAPTERS)[name]
    return IP.plus_geometry(cfg, E), cfg.cross_attention_dim, IP.plus_encoder_config(cfg, E).num_positions


def _plus(cfg, key="plus-test"):
    from cfgpp_b200 import ip_adapter as IP
    return IP.IPAdapter(key, dev, cfg, image_proj="resampler")


def _hidden(ad, B, seed=11):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, ad.resampler["seq_len"], ad.embed_dim, generator=g).half().to(dev)


def _bind_plus(net, B, h, w, uc, c, add, hidden=None):
    _bind(net, B, h, w, uc, c, add)
    if hidden is not None:
        net.set_ip_image_embeds(hidden)


# ---------------------------------------------------------------------------------------------------------------
# vision tower: hidden_states[num_layers - skip]
# ---------------------------------------------------------------------------------------------------------------
def _hidden_case(cfg, B, tol, seed=3):
    transformers = pytest.importorskip("transformers")
    from helpers import rel_l2
    from cfgpp_b200 import vision_encoder as V
    sd = V.synthetic_state_dict(cfg, seed=seed, device=dev)
    enc = V.NativeCLIPVisionEncoder(cfg, sd, dev)
    px = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(seed)).to(dev)
    tc = transformers.CLIPVisionConfig(hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                                       num_hidden_layers=cfg.num_hidden_layers,
                                       num_attention_heads=cfg.num_attention_heads, image_size=cfg.image_size,
                                       patch_size=cfg.patch_size, hidden_act=cfg.hidden_act,
                                       projection_dim=cfg.projection_dim, layer_norm_eps=cfg.layer_norm_eps)
    m = transformers.CLIPVisionModelWithProjection(tc).to(dev).eval()
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    with torch.no_grad():
        hs = m(pixel_values=px.half().float(), output_hidden_states=True).hidden_states
    for skip, ref in ((1, hs[-2]), (0, hs[-1]), (cfg.num_hidden_layers, hs[0])):
        got = enc.encode_hidden(px, skip=skip).float()
        err = rel_l2(got, ref)
        print(f"vision tower {cfg.hidden_size}x{cfg.num_hidden_layers} B{B} skip {skip}: hidden states rel-L2 vs fp32 "
              f"{err:.3e}")
        assert got.shape == ref.shape and torch.isfinite(got).all() and err <= tol
    enc.close()


def test_encode_hidden_tiny():
    from cfgpp_b200 import vision_encoder as V
    for B in (1, 3):
        _hidden_case(V.tiny_vision_config(), B, 2e-3)


def test_encode_hidden_vit_h():
    from cfgpp_b200 import vision_encoder as V
    _hidden_case(V.vit_h_config(), 2, 1e-2)


# ---------------------------------------------------------------------------------------------------------------
# the LayerNorm-concat kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NB", [1, 2, 16])
@pytest.mark.parametrize("C", [768, 1280])
def test_ln_concat_kernel(NB, C):
    """Every row of kv and q is bit-identical to layernorm_kernel on its segment and within ln_check's fp64 bound,
    with row means up to 100σ; rows land at (b, j) of kv and (b, i) of q exactly."""
    from cfgpp_b200 import _native as nv
    from test_gpu_norms import ln_check, ln_inputs
    from test_gpu_gemm import gen
    g = gen(1000 * NB + C)
    T, Q = P.vision_config("vit_h").num_positions, 16
    x, g0, b0 = ln_inputs(g, NB * T, C, 100.0, const_every=7)
    lat, g1, b1 = ln_inputs(g, NB * Q, C, 100.0)
    x, lat = x.reshape(NB, T, C), lat.reshape(NB, Q, C)
    kv, q = nv.op_ip_ln_concat(x, lat, g0, b0, g1, b1)
    want_x = ln_check(f"ln_concat LN0 NB{NB} C{C}", x.reshape(-1, C), g0, b0).reshape(NB, T, C)
    want_l = ln_check(f"ln_concat LN1 NB{NB} C{C}", lat.reshape(-1, C), g1, b1).reshape(NB, Q, C)
    bits = lambda t: t.view(torch.int16)  # noqa: E731
    assert torch.equal(bits(kv[:, :T]), bits(want_x)), "LN0 rows differ from layernorm_kernel"
    assert torch.equal(bits(kv[:, T:]), bits(want_l)), "LN1 rows in kv differ from layernorm_kernel"
    assert torch.equal(bits(q), bits(want_l)), "LN1 rows in q differ from layernorm_kernel"
    print(f"ln_concat NB{NB} C{C}: {NB * (T + Q)} rows bit-identical to layernorm_kernel")


# ---------------------------------------------------------------------------------------------------------------
# the Resampler's attention and LayerNorms at the production sizes, under the existing per-element gates (its GEMMs
# run in test_gpu_gemm.py's production lists)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NB", P.IP_PLUS_NB)
@pytest.mark.parametrize("name", [m for m, _ in P.IP_PLUS_ADAPTERS])
def test_resampler_production_launches(name, NB):
    from test_gpu_attention import check
    from test_gpu_gemm import gen
    from test_gpu_norms import ln_check, ln_inputs
    geo, D, T = _geometry(name)
    Q, H, dim = geo["num_queries"], geo["heads"], geo["dim"]
    inner = 64 * H
    g = gen(NB * 7 + H)
    q = torch.randn(NB, Q, inner, generator=g, device=dev).half()
    kvb = torch.randn(NB, T + Q, 2 * inner, generator=g, device=dev).half()
    check(f"{name} plus NB{NB} sdpa", q, kvb[..., :inner], kvb[..., inner:], H, 64)
    for M, C in ((NB * Q, dim), (NB * Q, D)):
        ln_check(f"{name} plus NB{NB} layernorm {M}x{C}", *ln_inputs(g, M, C, 10.0))


# ---------------------------------------------------------------------------------------------------------------
# the Resampler's tokens against the oracle
# ---------------------------------------------------------------------------------------------------------------
def native_tokens(net):
    """The image tokens of the last set_ip_image_embeds, [2 * batch * Q, D] fp16 (the projection is run again)."""
    from cfgpp_b200 import _native as nv
    out = torch.empty(2 * net.batch * net.ip_adapter.n_tokens, net.cfg.cross_attention_dim, dtype=torch.float16,
                      device=dev)
    nv.check(net.lib.cfgpp_dbg_ip_image_proj(net._h, nv.ptr(out), nv.stream_ptr()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name,batches", [("tiny_sd15", (1, 3)), ("tiny_sdxl", (2,)), ("sd15", (1, 8)),
                                          ("sdxl", (1, 8))])
def test_resampler_tokens_against_the_oracle(name, batches):
    """The native Resampler's tokens (tiny geometry; SD v1.5 Plus: dim 768, 12 heads; SDXL Plus vit-h: dim 1280,
    20 heads, D 2048; depth 4, 16 queries, 257 x 1280 hidden states) against the oracle on the same fp16 weights:
    rel-L2 <= 5e-3 against the fp16 oracle, and the error against the fp32 oracle at most 1.5x the fp16 oracle's own.
    Every row of the batch, the unconditional half included."""
    from helpers import rel_l2
    cfg, sd, net = _net(name)
    ad = _plus(cfg)
    ad._uncond = _hidden(ad, 1, seed=12)
    g = ad.resampler
    w = {k: v for k, v in ad.weights.items() if k.startswith("image_proj.")}
    net.attach_ip_adapter(ad)
    hw = 32 if name.startswith("tiny") else 64
    for B in batches:
        hidden = _hidden(ad, B, seed=20 + B)
        net.prepare(B, hw, hw)
        net.set_ip_image_embeds(hidden)
        got = native_tokens(net).float().reshape(2 * B, g["num_queries"], -1)
        rows = ad.image_rows(hidden)
        refs = {}
        with torch.no_grad():
            for dt in (torch.float16, torch.float32):
                refs[dt] = PO.resampler({k: v.to(dev, dt) for k, v in w.items()}, rows.to(dt), g["heads"],
                                        g["depth"]).float()
        r16, r32 = refs[torch.float16], refs[torch.float32]
        e16, e32, e_ref = rel_l2(got, r16), rel_l2(got, r32), rel_l2(r16, r32)
        print(f"plus tokens {name} B{B}: rel-L2 vs fp16 oracle {e16:.3e}, vs fp32 {e32:.3e} "
              f"(fp16 oracle vs fp32 {e_ref:.3e})")
        assert torch.isfinite(got).all()
        assert e16 <= 5e-3
        assert e32 <= 1.5 * e_ref
    net.close()


def test_reloaded_weight_of_another_shape_is_refused():
    """A Resampler weight loaded again after attach with another shape is refused, naming it, when the plan is built;
    loading the right shape again restores the adapter."""
    import ctypes
    from ctypes import c_int
    from cfgpp_b200 import _native as nv
    from cfgpp_b200._native import NativeError
    cfg, sd, net = _net("tiny_sd15")
    ad = _plus(cfg)
    ad._uncond = _hidden(ad, 1, seed=12)
    B, hw = 1, 32
    net.attach_ip_adapter(ad)
    net.prepare(B, hw, hw)
    hidden = _hidden(ad, B)
    net.set_ip_image_embeds(hidden)
    want = native_tokens(net)

    def load(key, t):
        t = t.to(dev).contiguous()
        shape = (ctypes.c_int64 * t.dim())(*t.shape)
        nv.check(net.lib.cfgpp_ip_adapter_load_weight(net._h, key.encode(), nv.ptr(t), shape, c_int(t.dim()),
                                                      c_int(nv.dtype_code(t)), nv.stream_ptr()))
        torch.cuda.synchronize()

    rows = ad.image_rows(hidden).to(dev)
    for key in ("image_proj.layers.0.0.to_q.weight", "image_proj.latents"):
        good = ad.weights[key]
        load(key, good[:, :8] if key.endswith("latents") else good[:64])
        with pytest.raises(NativeError, match=key.replace(".", r"\.") + ": shape"):
            nv.check(net.lib.cfgpp_prepare(net._h, c_int(B), c_int(hw), c_int(hw)))
        with pytest.raises(NativeError, match="cfgpp_prepare"):
            nv.check(net.lib.cfgpp_set_ip_image_hidden_states(net._h, nv.ptr(rows), nv.stream_ptr()))
        load(key, good)
        nv.check(net.lib.cfgpp_prepare(net._h, c_int(B), c_int(hw), c_int(hw)))
        nv.check(net.lib.cfgpp_set_ip_image_hidden_states(net._h, nv.ptr(rows), nv.stream_ptr()))
        got = torch.empty_like(want)
        nv.check(net.lib.cfgpp_dbg_ip_image_proj(net._h, nv.ptr(got), nv.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(got, want)
    net.close()


# ---------------------------------------------------------------------------------------------------------------
# the Plus adapter in the UNet executor
# ---------------------------------------------------------------------------------------------------------------
def plus_forward_case(name, B, h, w, t, scale=0.7):
    import controlnet_oracle as CO
    from helpers import rel_l2
    from oracle import unet as O
    from cfgpp_b200 import ip_adapter as IP
    cfg, sd, net = _net(name)
    ad = _plus(cfg)
    z, uc, c, add, _ = _inputs(cfg, B, h, w, 8)
    hidden = _hidden(ad, B)
    uncond = _hidden(ad, 1, seed=12)
    ad._uncond = uncond  # the zero-image features are the encoder's business; pin them here
    net.attach_ip_adapter(ad)
    _bind_plus(net, B, h, w, uc, c, add, hidden)
    net.set_ip_adapter_scale(scale)
    got = _native(net, z, t)
    net.attach_ip_adapter(None)
    _bind(net, B, h, w, uc, c, add)
    plain = _native(net, z, t)
    net.close()
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
    refs = {}
    for dtype in (torch.float16, torch.float32):
        um = O.build_unet(CO.oracle_cfg(cfg), sd, dtype=dtype, device=dev)
        st = PO.attach(um, ad.weights, IP.attn2_blocks(cfg), ad.resampler)
        st["scale"] = scale
        a = {k: v.to(dtype) for k, v in add.items()} if add else None
        with torch.autocast("cuda", dtype=torch.float16, enabled=dtype == torch.float16), torch.no_grad():
            PO.set_hidden_states(st, hidden.to(dtype), uncond.to(dtype))
            refs[dtype] = CO.unet_forward(um, z_in, t_in, ctx.to(dtype), a)["sample"].float()
        del um
    r16, r32 = refs[torch.float16], refs[torch.float32]
    e16, e_ref, e_plain = rel_l2(got, r16), rel_l2(r16, r32), rel_l2(plain, got)
    print(f"plus {name} {B}x{h}x{w}: rel-L2 vs fp16 oracle {e16:.3e}, vs fp32 {rel_l2(got, r32):.3e} "
          f"(fp16 oracle vs fp32 {e_ref:.3e}); with vs without the adapter {e_plain:.3e}")
    assert torch.isfinite(got).all()
    assert e16 <= TOL
    assert rel_l2(got, r32) <= 1.5 * e_ref + 1e-4
    assert e_plain >= 10 * TOL


@pytest.mark.parametrize("name,B,h,w,t", [("tiny_sd15", 1, 32, 32, 401), ("tiny_sd15", 2, 16, 32, 301),
                                          ("tiny_sdxl", 2, 32, 32, 999)])
def test_plus_forward_tiny(name, B, h, w, t):
    plus_forward_case(name, B, h, w, t)


@pytest.mark.parametrize("name,hw", [("sd15", 64), ("sdxl", 128)])
def test_plus_forward_full_size(name, hw):
    plus_forward_case(name, 1, hw, hw, 501)


def test_plus_trajectory_scale_zero_callback_and_scale_word():
    """At s = 0 the fused trajectory with a Plus adapter equals the adapter-free one bit for bit; the fused trajectory
    equals the callback path; a scale change never recaptures the step graph."""
    cfg, sd, net = _net("tiny_sdxl")
    ad = _plus(cfg)
    ad._uncond = _hidden(ad, 1, seed=12)
    B, h, w = 2, 32, 32
    z, uc, c, add, _ = _inputs(cfg, B, h, w, 8)
    hidden = _hidden(ad, B)
    _bind(net, B, h, w, uc, c, add)
    plain, _ = _trajectory(net, z)
    net.attach_ip_adapter(ad)
    _bind_plus(net, B, h, w, uc, c, add, hidden)
    net.set_ip_adapter_scale(0.0)
    assert torch.equal(_trajectory(net, z)[0], plain), "s = 0 differs from the trajectory without an adapter"
    n0 = _captures(net)
    net.set_ip_adapter_scale(0.8)
    z08, steps = _trajectory(net, z)
    assert _captures(net) == n0, "setting the scale recaptured the step graph"
    assert not torch.equal(z08, plain)
    net.set_state(z)
    for i, st in enumerate(steps):
        _, zt = net.callback_step(i, st)
    assert torch.equal(zt, z08), "fused trajectory != callback path"
    net.close()


def test_plain_plus_plain_on_one_handle_and_refusals():
    """plain -> Plus -> plain on one live handle equals fresh handles bit for bit; each setter refuses the other kind
    of adapter; attach_resampler names a weight that does not fit."""
    from ctypes import c_int
    from cfgpp_b200 import _native as nv, ip_adapter as IP
    from cfgpp_b200._native import NativeError
    name, B, h, w = "tiny_sd15", 1, 32, 32
    cfg, sd, net = _net(name)
    plain_ad, plus_ad = IP.IPAdapter("ip-a", dev, cfg), _plus(cfg)
    plus_ad._uncond = _hidden(plus_ad, 1, seed=12)
    z, uc, c, add, embeds = _inputs(cfg, B, h, w, plain_ad.embed_dim)
    hidden = _hidden(plus_ad, B)
    outs = []
    for ad, e in ((plain_ad, embeds), (plus_ad, hidden), (plain_ad, embeds)):
        net.attach_ip_adapter(ad)
        _bind(net, B, h, w, uc, c, add, None)
        net.set_ip_image_embeds(e)
        outs.append(_native(net, z, 501))
    with pytest.raises(NativeError, match="cfgpp_set_ip_image_embeds"):
        nv.check(net.lib.cfgpp_set_ip_image_hidden_states(net._h, nv.ptr(torch.cat([hidden, hidden])), nv.stream_ptr()))
    net.attach_ip_adapter(plus_ad)
    _bind(net, B, h, w, uc, c, add, None)
    with pytest.raises(NativeError, match="cfgpp_set_ip_image_hidden_states"):
        nv.check(net.lib.cfgpp_set_ip_image_embeds(net._h, nv.ptr(torch.cat([embeds, embeds])), nv.stream_ptr()))
    r = plus_ad.resampler
    bad = (c_int * 7)(r["num_queries"], r["embed_dim"], r["seq_len"], r["dim"], r["heads"] + 1, r["depth"], r["ff_mult"])
    with pytest.raises(NativeError, match=r"image_proj\.layers\.0\.0\.to_q\.weight: shape"):
        nv.check(net.lib.cfgpp_ip_adapter_attach_resampler(net._h, bad))
    net.close()
    for i, (ad, e) in enumerate(((plain_ad, embeds), (plus_ad, hidden))):
        _, _, fresh = _net(name)
        fresh.attach_ip_adapter(ad)
        _bind(fresh, B, h, w, uc, c, add, None)
        fresh.set_ip_image_embeds(e)
        want = _native(fresh, z, 501)
        fresh.close()
        assert torch.equal(outs[i], want), f"step {i} differs from a fresh handle"
        if i == 0:
            assert torch.equal(outs[2], want), "plain after Plus differs from a fresh handle"
    assert not torch.equal(outs[0], outs[1])


def test_plus_batch_equals_single_runs():
    """A batch of B prompts with B reference images equals B single-image runs."""
    from helpers import rel_l2
    cfg, sd, net = _net("tiny_sd15")
    ad = _plus(cfg)
    ad._uncond = _hidden(ad, 1, seed=12)
    B, h, w = 3, 32, 32
    z, uc, c, add, _ = _inputs(cfg, B, h, w, 8)
    hidden = _hidden(ad, B)
    net.attach_ip_adapter(ad)
    _bind_plus(net, B, h, w, uc, c, add, hidden)
    both = _native(net, z, 501)
    for b in range(B):
        _bind_plus(net, 1, h, w, uc[b:b + 1], c[b:b + 1], add, hidden[b:b + 1])
        one = _native(net, z[b:b + 1], 501)
        for half in range(2):
            err = rel_l2(one[half:half + 1], both[half * B + b:half * B + b + 1])
            print(f"plus batch row {b} half {half}: rel-L2 vs the single run {err:.3e}")
            assert err <= 2e-3
    net.close()


@pytest.mark.parametrize("family", ["sd", "sdxl"])
def test_solver_sample_with_plus(family):
    """sample(ip_adapter=Plus) end to end on tiny UNets with the tiny tower: the fused and callback paths give the same
    image, the adapter moves the image, scale 0 is the plain image bit for bit, it composes with a ControlNet, and a
    later call without it is the plain image again."""
    from types import SimpleNamespace
    from helpers import rel_l2
    from cfgpp_b200 import config as C, controlnet as CN, latent_diffusion as LD, latent_sdxl as LX, weights as Wt
    from test_gpu_controlnet import _LatentVAE
    cfg = C.tiny_sd15_config() if family == "sd" else C.tiny_sdxl_config()
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    vae = _LatentVAE()
    s = (LD if family == "sd" else LX).get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=6),
                                                   device=dev, unet_config=cfg, state_dict=sd, vae=vae)
    hw = cfg.sample_size
    g = torch.Generator().manual_seed(4)
    zT = torch.randn(2, 4, hw, hw, generator=g)
    img = (torch.rand(48, 40, 3, generator=g) * 255).to(torch.uint8).numpy()
    ad = _plus(cfg, "plus-solver")

    def run(**kw):
        if family == "sd":
            s.sample(cfg_guidance=0.6, prompt=["", ["a cat", "a dog"]], zT=zT, **kw)
        else:
            s.sample(prompt1=["", ["a cat", "a dog"]], prompt2=["", ["a cat", "a dog"]], cfg_guidance=0.6,
                     target_size=(8 * hw, 8 * hw), zT=zT, **kw)
        return vae.latents[-1].float()

    plain = run()
    fused = run(ip_adapter=ad, ip_adapter_image=img, ip_adapter_scale=0.8)
    e_plain = rel_l2(fused, plain)
    print(f"plus sample {family}: with vs without the adapter {e_plain:.3e}")
    assert e_plain >= 1e-2
    assert torch.equal(run(ip_adapter=ad, ip_adapter_image=img, ip_adapter_scale=0.8, callback_fn=lambda i, t, kw: kw),
                       fused)
    assert torch.equal(run(ip_adapter=ad, ip_adapter_image=img, ip_adapter_scale=0.0), plain)
    cn = CN.ControlNet("synthetic-controlnet", dev, base_cfg=cfg)
    both = run(ip_adapter=ad, ip_adapter_image=img, ip_adapter_scale=0.8, controlnet=cn,
               control_image=torch.rand(1, 3, 8 * hw, 8 * hw, generator=g))
    print(f"plus sample {family} + ControlNet: vs Plus alone {rel_l2(both, fused):.3e}")
    assert torch.isfinite(both).all() and rel_l2(both, fused) >= 1e-2
    assert torch.equal(run(), plain) and s.unet.ip_adapter is None
