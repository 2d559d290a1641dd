"""IP-Adapter on the GPU: the decoupled cross-attention kernel `attn_ip_kernel<HD>` (`attention.cu`) through
`cfgpp_op_attention_ip`, and the adapter inside the UNet executor.

Kernel gate. The reference is fp64 on the same fp16 inputs: ref = ref1 + s·ref2, ref1 the softmax attention over the
text tokens, ref2 over the image tokens. The kernel forms O1/l1 and O2/l2 in fp32 with the plain kernel's rounding
points and rounds their sum once, so the per-element bound is
    E = (E1 − ½ulp(ref1)) + |s|·(E2 − ½ulp(ref2)) + 2^-23·(|ref1| + |s|·|ref2|) + ½ulp(ref)
with E1 / E2 the bounds of `test_gpu_attention._reference` for each segment (each of which carries its own ½ulp of a
final rounding that the fused kernel does not do), the fp32 rounding of the product s·y2 and of the sum, and the one
fp16 rounding. The scale is read from the middle word of [7, s, −3], so a kernel that reads a neighbouring word fails.

The image families cover a flat and a peaked image softmax and image logits about 40 nats below or above the text
logits: a kernel that shares the running max between the segments underflows one of the two sums there."""
import math

import pytest
import torch

from test_gpu_attention import _reference, family, fused, gen, heads, padded, ulp16

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

HEAD_DIMS = (64, 40, 80, 160)
NKV2 = (1, 4, 16, 63, 64)
SCALES = (0.0, 0.5, 1.0, 2.0)
IMAGE_FAMILIES = ("flat", "peaked", "far_below", "far_above")


def scale_word(s):
    """A device tensor [7, s, −3]; the kernel is handed the middle word."""
    return torch.tensor([7.0, s, -3.0], dtype=torch.float32, device=dev)[1:2]


def image_tokens(name, g, B, Nkv2, H, hd, u):
    """k2 / v2 [B, Nkv2, H, hd] fp32 of one image family. The query rows of `check_ip` carry the direction u
    (|u|² = hd), so k2 += γ·u moves every image logit by about γ·sqrt(hd)."""
    k2 = torch.randn(B, Nkv2, H, hd, generator=g, device=dev)
    v2 = torch.randn(B, Nkv2, H, hd, generator=g, device=dev)
    if name == "flat":
        return 1.2 * k2, v2
    if name == "peaked":
        return 3 * k2, v2
    if name == "far_below":
        return k2 - (40 / math.sqrt(hd)) * u, v2
    if name == "far_above":
        return k2 + (40 / math.sqrt(hd)) * u, v2
    raise ValueError(name)


def attention_ip(q, k, v, k2, v2, s, H, hd):
    from cfgpp_b200 import _native as nv
    return nv.op_attention_ip(q, k, v, k2, v2, scale_word(s), H, head_dim=hd)


def check_ip(what, q, k, v, k2, v2, s, H, hd):
    """Run the fused kernel and gate every element against the fp64 reference. Returns the output."""
    out = attention_ip(q, k, v, k2, v2, s, H, hd)
    B, Nq, C = q.shape
    Nkv, Nkv2, hdp = k.shape[1], k2.shape[1], C // H
    o = out.unflatten(2, (H, hdp))
    assert torch.isfinite(o).all(), f"{what}: non-finite output"
    if hdp > hd:
        assert (o[..., hd:].view(torch.int16) == 0).all(), f"{what}: padding columns are not +0"
    qh, kh, vh, k2h, v2h = (t.unflatten(2, (H, hdp))[..., :hd] for t in (q, k, v, k2, v2))
    worst = torch.zeros((), dtype=torch.float64, device=dev)
    for b in range(B):
        Q = qh[b].transpose(0, 1).double()
        r1, e1 = _reference(Q, kh[b].transpose(0, 1).double(), vh[b].transpose(0, 1).double(), hdp)
        r2, e2 = _reference(Q, k2h[b].transpose(0, 1).double(), v2h[b].transpose(0, 1).double(), hdp)
        ref = r1 + s * r2
        bound = ((e1 - 0.5 * ulp16(r1)) + abs(s) * (e2 - 0.5 * ulp16(r2))
                 + 2.0 ** -23 * (r1.abs() + abs(s) * r2.abs()) + 0.5 * ulp16(ref))
        d = o[b, :, :, :hd].transpose(0, 1).double() - ref
        worst = torch.maximum(worst, (d.abs() / bound).max())
    worst = worst.item()
    assert worst <= 1.0, f"{what}: error {worst:.3f}x the bound"
    return out


@pytest.mark.parametrize("hd", HEAD_DIMS)
@pytest.mark.parametrize("image", IMAGE_FAMILIES)
def test_fused_kernel_sweep(image, hd):
    """Every Nkv2 in 1, 4, 16, 63, 64 and s in 0, 0.5, 1, 2, against text segments of one and three KV tiles (77 and
    150 tokens) with flat and peaked softmaxes, one and three query tiles; k2 / v2 are slices of one fused buffer as
    the UNet's image K‖V projection writes them. At s = 0 the output is the plain kernel's bit for bit."""
    from cfgpp_b200 import _native as nv
    B, H, hdp = 2, 2, padded(hd)
    g = gen(IMAGE_FAMILIES.index(image) * 1000 + hd + 5)
    u = torch.randint(0, 2, (H, hd), generator=g, device=dev).float() * 2 - 1
    worst = 0
    for text in ("flat", "peaked"):
        for Nq in (1, 130):
            for Nkv in (77, 150):
                q, k, v = family(text, g, B, Nq, Nkv, H, hd)
                q = heads(q + u, hdp)
                k, v = fused(heads(k, hdp), heads(v, hdp))
                plain = nv.op_attention(q, k, v, H, head_dim=hd)
                for Nkv2 in NKV2:
                    k2, v2 = fused(*(heads(t, hdp) for t in image_tokens(image, g, B, Nkv2, H, hd, u)))
                    for s in SCALES:
                        what = f"{text}/{image} hd{hd} {Nq}x{Nkv}+{Nkv2} s={s}"
                        out = check_ip(what, q, k, v, k2, v2, s, H, hd)
                        if s == 0:
                            assert torch.equal(out, plain), f"{what}: s = 0 differs from the plain kernel"
                        worst += 1
    assert worst == 2 * 2 * 2 * len(NKV2) * len(SCALES)


def _attn2_cases():
    """The distinct cross-attention launch shapes of SD v1.5 512² and SDXL 1024² / 1216x832 (`production.py`), with
    the plain adapter's IP_TOKENS image tokens and the Plus adapter's num_queries (`ip_adapter.plus_geometry`)."""
    import production as P
    from cfgpp_b200 import config as C, ip_adapter as IP
    seen, cases = set(), []
    for n_img in (P.IP_TOKENS, IP.plus_geometry(C.CONFIGS["sd15"](), 1280)["num_queries"]):
        for m, h, w in P.unet_sizes():
            if m not in ("sd15", "sdxl"):
                continue
            for l in P.unet_attn_launches(C.CONFIGS[m](), h, w):
                shape = (l["heads"], l["Nq"], l["hd"], n_img)
                if l["name"].endswith("attn2.sdpa") and shape not in seen:
                    seen.add(shape)
                    tag = f"{P.size_tag(m, h, w)}-H{shape[0]}-{shape[1]}-hd{shape[2]}"
                    cases.append(pytest.param(*shape, id=tag if n_img == P.IP_TOKENS else f"{tag}-img{n_img}"))
    return cases


@pytest.mark.parametrize("H,Nq,hd,n_img", _attn2_cases())
@pytest.mark.parametrize("s", [0.5, 1.0])
def test_production_attn2_shapes(H, Nq, hd, n_img, s):
    """Every attn2 launch of SD v1.5 512² and SDXL 1024² / 1216x832 at UNet batch 4 with 4 image tokens (the plain
    adapter) and 16 (IP-Adapter Plus), peaked text and image softmaxes, in the UNet's layouts: q from its own buffer,
    K / V and K2 / V2 column slices of the prompt's and the image's K‖V buffers."""
    NB, hdp = 4, padded(hd)
    g = gen(Nq * 31 + H * 7 + hd + int(4 * s) + 1000 * (n_img - 4))  # the 4-token cases keep their inputs
    q, k, v = family("peaked", g, NB, Nq, 77, H, hd)
    u = torch.zeros(H, hd, device=dev)
    k2, v2 = image_tokens("peaked", g, NB, n_img, H, hd, u)
    k, v = fused(heads(k, hdp), heads(v, hdp))
    k2, v2 = fused(heads(k2, hdp), heads(v2, hdp))
    check_ip(f"NB{NB} H{H} {Nq}x77+{n_img} hd{hd} s={s}", heads(q, hdp), k, v, k2, v2, s, H, hd)


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_known_answer_and_scale_linearity(hd):
    """Identical image keys: every image p is 1 and O2/l2 is the shared value row w0 exactly, so the output is
    fp16(y1 + s·w0) with y1 the plain kernel's fp32 result. With w0 = 0 it is the plain kernel's output for every s;
    with text and image tokens equal (same k, v rows twice), the image segment repeats the text one and s = 1 gives
    fp16(2·y1), which is the plain kernel's output on 2·v (a power of two scales every fp32 step exactly)."""
    from cfgpp_b200 import _native as nv
    B, H, Nq, Nkv, hdp = 2, 2, 130, 40, padded(hd)
    g = gen(hd + 21)
    q, k, v = (heads(t, hdp) for t in family("flat", g, B, Nq, Nkv, H, hd))
    plain = nv.op_attention(q, k, v, H, head_dim=hd)
    k0 = heads(torch.randn(B, 1, H, hd, generator=g, device=dev).expand(B, 4, H, hd), hdp)
    zero = torch.zeros_like(k0)
    for s in SCALES:
        assert torch.equal(attention_ip(q, k, v, k0, zero, s, H, hd), plain), f"hd{hd} s={s}: zero image values"
    assert torch.equal(attention_ip(q, k, v, k, v, 1.0, H, hd), nv.op_attention(q, k, v * 2, H, head_dim=hd)), \
        f"hd{hd}: doubled segment"


# ---------------------------------------------------------------------------------------------------------------
# the adapter in the UNet executor
# Tolerance of the forward comparisons: test_gpu_unet.py's (rel-L2 <= 5e-3 against the fp16-autocast oracle, and at
# most 1.5x that oracle's own error against the fp32 oracle).
# ---------------------------------------------------------------------------------------------------------------
TOL = 5e-3


def _net(name, seed=1234):
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg = C.CONFIGS[name]()
    sd = Wt.synthetic_state_dict(cfg, seed=seed, device=dev)
    return cfg, sd, NativeUNet(cfg, sd, dev)


def _adapter(cfg, key="ip-test"):
    from cfgpp_b200 import ip_adapter as IP
    return IP.IPAdapter(key, dev, cfg)


def _inputs(cfg, B, h, w, E, seed=5):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 4, h, w, generator=g).to(dev)
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    add = None
    if cfg.addition_embed_type == "text_time":
        add = {"text_embeds": torch.randn(2 * B, cfg.pooled_dim, generator=g).half().to(dev),
               "time_ids": torch.tensor([[8. * h, 8. * w, 0, 0, 8. * h, 8. * w]] * (2 * B)).half().to(dev)}
    embeds = torch.randn(B, E, generator=g).half().to(dev)
    return z, uc, c, add, embeds


def _bind(net, B, h, w, uc, c, add, embeds=None):
    net.prepare(B, h, w)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"] if add else None, add["time_ids"].float() if add else None)
    if embeds is not None:
        net.set_ip_image_embeds(embeds)


def _native(net, z, t):
    eu, ec = net.predict_noise(z, float(t))
    return torch.cat([eu, ec]).float()


def forward_case(name, B, h, w, t, scale=0.7):
    import controlnet_oracle as CO
    import ip_adapter_oracle as IO
    from helpers import rel_l2
    from oracle import unet as O
    from cfgpp_b200 import ip_adapter as IP
    cfg, sd, net = _net(name)
    ad = _adapter(cfg)
    z, uc, c, add, embeds = _inputs(cfg, B, h, w, ad.embed_dim)
    net.attach_ip_adapter(ad)
    _bind(net, B, h, w, uc, c, add, embeds)
    net.set_ip_adapter_scale(scale)
    got = _native(net, z, t)
    net.attach_ip_adapter(None)
    _bind(net, B, h, w, uc, c, add)
    plain = _native(net, z, t)
    net.close()
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
    blocks = IP.attn2_blocks(cfg)
    refs = {}
    for dtype in (torch.float16, torch.float32):
        um = O.build_unet(CO.oracle_cfg(cfg), sd, dtype=dtype, device=dev)
        st = IO.attach(um, ad.weights, blocks, ad.n_tokens, cfg.cross_attention_dim)
        st["scale"] = scale
        a = {k: v.to(dtype) for k, v in add.items()} if add else None
        with torch.autocast("cuda", dtype=torch.float16, enabled=dtype == torch.float16), torch.no_grad():
            IO.set_embeds(st, embeds.to(dtype))
            refs[dtype] = CO.unet_forward(um, z_in, t_in, ctx.to(dtype), a)["sample"].float()
        del um
    r16, r32 = refs[torch.float16], refs[torch.float32]
    e16, e_ref, e_plain = rel_l2(got, r16), rel_l2(r16, r32), rel_l2(plain, got)
    print(f"{name} {B}x{h}x{w}: rel-L2 vs fp16 oracle {e16:.3e}, vs fp32 {rel_l2(got, r32):.3e} "
          f"(fp16 oracle vs fp32 {e_ref:.3e}); with vs without the adapter {e_plain:.3e}")
    assert torch.isfinite(got).all()
    assert e16 <= TOL
    assert rel_l2(got, r32) <= 1.5 * e_ref + 1e-4
    assert e_plain >= 10 * TOL  # the image segment matters: a skipped one cannot pass


@pytest.mark.parametrize("name,B,h,w,t", [("tiny_sd15", 1, 32, 32, 401), ("tiny_sd15", 2, 16, 32, 301),
                                          ("tiny_sdxl", 1, 32, 32, 601), ("tiny_sdxl", 2, 32, 32, 999)])
def test_ip_forward_tiny(name, B, h, w, t):
    forward_case(name, B, h, w, t)


@pytest.mark.parametrize("name,hw", [("sd15", 64), ("sdxl", 128)])
def test_ip_forward_full_size(name, hw):
    forward_case(name, 1, hw, hw, 501)


def _trajectory(net, z, nfe=4, lam=0.6):
    from cfgpp_b200 import schedule as S
    steps = S.ddim_cfgpp_steps(S.Schedule.make(nfe), lam, True)
    return net.run_trajectory(S.STEP_DDIM_CFGPP, torch.float32, steps, z)[1], steps


def _captures(net):
    from ctypes import byref, c_int
    from cfgpp_b200 import _native as nv
    n = c_int()
    nv.check(net.lib.cfgpp_dbg_graph_captures(net._h, byref(n)))
    return n.value


def test_scale_zero_clear_and_scale_word():
    """A whole fused trajectory with an adapter at s = 0 equals the trajectory without one bit for bit; so does the
    trajectory after clearing the adapter. Changing s between trajectories changes the output without capturing the
    step graph again, and the fused trajectory equals the callback path (predict_noise + apply_step) bit for bit."""
    cfg, sd, net = _net("tiny_sdxl")
    ad = _adapter(cfg)
    B, h, w = 2, 32, 32
    z, uc, c, add, embeds = _inputs(cfg, B, h, w, ad.embed_dim)
    _bind(net, B, h, w, uc, c, add)
    plain, _ = _trajectory(net, z)
    net.attach_ip_adapter(ad)
    _bind(net, B, h, w, uc, c, add, embeds)
    net.set_ip_adapter_scale(0.0)
    assert torch.equal(_trajectory(net, z)[0], plain), "s = 0 differs from the trajectory without an adapter"
    n0 = _captures(net)
    net.set_ip_adapter_scale(0.8)
    z08, steps = _trajectory(net, z)
    assert _captures(net) == n0, "setting the scale recaptured the step graph"
    assert not torch.equal(z08, plain)
    net.set_ip_adapter_scale(0.4)
    z04, _ = _trajectory(net, z)
    assert _captures(net) == n0 and not torch.equal(z04, z08)
    net.set_ip_adapter_scale(0.8)
    assert torch.equal(_trajectory(net, z)[0], z08)
    net.set_state(z)  # the callback path of the same schedule
    for i, st in enumerate(steps):
        _, zt = net.callback_step(i, st)
    assert torch.equal(zt, z08), "fused trajectory != callback path"
    net.attach_ip_adapter(None)
    _bind(net, B, h, w, uc, c, add)
    assert torch.equal(_trajectory(net, z)[0], plain), "attach -> clear does not restore the plain trajectory"
    net.close()


def test_new_image_same_prompt_reprojects_and_batching():
    """Binding another reference image with the same prompt projects it again; a batch of B prompts with B images
    equals B single-image runs (the image tokens of row b only reach row b)."""
    cfg, sd, net = _net("tiny_sd15")
    ad = _adapter(cfg)
    B, h, w = 3, 32, 32
    z, uc, c, add, embeds = _inputs(cfg, B, h, w, ad.embed_dim)
    net.attach_ip_adapter(ad)
    _bind(net, B, h, w, uc, c, add, embeds)
    both = _native(net, z, 501)
    net.set_ip_image_embeds(embeds.flip(0))
    flipped = _native(net, z, 501)
    assert not torch.equal(both, flipped)
    net.set_ip_image_embeds(embeds)
    assert torch.equal(_native(net, z, 501), both)
    for b in range(B):
        _bind(net, 1, h, w, uc[b:b + 1], c[b:b + 1], add, embeds[b:b + 1])
        one = _native(net, z[b:b + 1], 501)
        from helpers import rel_l2
        for half in range(2):
            got, want = one[half:half + 1], both[half * B + b:half * B + b + 1]
            assert rel_l2(got, want) <= 2e-3, f"image {b}, half {half}"
    net.close()


@pytest.mark.parametrize("name,hw", [("tiny_sd15", 32), ("tiny_sdxl", 32), ("sd15", 64)])
def test_second_adapter_on_a_live_handle(name, hw):
    """Attaching adapter B to a handle that already packed adapter A loads B's keys over A's and re-packs every image
    K‖V operand that reads them in place (a plain concatenation at head_dim 64, head-padded at SD v1.5's 40 / 80 /
    160): the forward equals a fresh handle's with B bit for bit."""
    cfg, sd, net = _net(name)
    a, b = _adapter(cfg, "ip-a"), _adapter(cfg, "ip-b")
    B, h, w = 1, hw, hw
    z, uc, c, add, embeds = _inputs(cfg, B, h, w, a.embed_dim)
    net.attach_ip_adapter(a)
    _bind(net, B, h, w, uc, c, add, embeds)
    with_a = _native(net, z, 501)
    net.attach_ip_adapter(b)
    _bind(net, B, h, w, uc, c, add, embeds)
    got = _native(net, z, 501)
    net.close()
    _, _, fresh = _net(name)
    fresh.attach_ip_adapter(b)
    _bind(fresh, B, h, w, uc, c, add, embeds)
    want = _native(fresh, z, 501)
    fresh.close()
    assert not torch.equal(got, with_a), "adapter B's forward equals adapter A's"
    assert torch.equal(got, want), "B loaded over A differs from B on a fresh handle"


def test_controlnet_handle_refuses_adapter_and_sees_text_only():
    """A ControlNet handle refuses an adapter; with both attached the forward matches the oracle ControlNet (text
    context only) feeding the oracle UNet with the adapter."""
    import controlnet_oracle as CO
    import ip_adapter_oracle as IO
    from helpers import rel_l2
    from oracle import unet as O
    from cfgpp_b200 import controlnet as CN, ip_adapter as IP
    from cfgpp_b200._native import NativeError
    cfg, sd, net = _net("tiny_sd15")
    cn_cfg = CN.controlnet_config(cfg)
    cn_sd = CN.synthetic_controlnet_state_dict(cn_cfg, seed=99, device=dev)
    cn = CN.NativeControlNet(cn_cfg, cn_sd, dev)
    with pytest.raises(NativeError, match="ControlNet"):
        from ctypes import c_int
        from cfgpp_b200 import _native as nv
        nv.check(cn.lib.cfgpp_ip_adapter_attach(cn._h, c_int(4), c_int(256)))
    ad = _adapter(cfg)
    B, h, w, t, scale = 1, 32, 32, 401, 0.7
    z, uc, c, add, embeds = _inputs(cfg, B, h, w, ad.embed_dim)
    image = torch.rand(B, 3, 8 * h, 8 * w, generator=torch.Generator().manual_seed(3)).to(dev)
    net.attach_controlnet(cn)
    net.attach_ip_adapter(ad)
    _bind(net, B, h, w, uc, c, add, embeds)
    net.set_control_image(image)
    got = _native(net, z, t)
    net.close()
    cn.close()
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
    um = O.build_unet(CO.oracle_cfg(cfg), sd, dtype=torch.float16, device=dev)
    cm = CO.build_controlnet(cn_cfg, cn_sd, dtype=torch.float16, device=dev)
    st = IO.attach(um, ad.weights, IP.attn2_blocks(cfg), ad.n_tokens, cfg.cross_attention_dim)
    with torch.autocast("cuda", dtype=torch.float16), torch.no_grad():
        IO.set_embeds(st, embeds)
        dres, mres = cm(z_in, t_in, ctx, torch.cat([image] * 2), 1.0, None)
        ref = CO.unet_forward(um, z_in, t_in, ctx, None, dres, mres)["sample"].float()
    assert rel_l2(got, ref) <= TOL


# ---------------------------------------------------------------------------------------------------------------
# CLIP vision tower against transformers' CLIPVisionModelWithProjection (fp32, the same seeded fp16 weights)
# ---------------------------------------------------------------------------------------------------------------
def _vision_case(cfg, B, final_tol, seed=3):
    transformers = pytest.importorskip("transformers")
    from helpers import rel_l2
    from cfgpp_b200 import vision_encoder as V
    sd = V.synthetic_state_dict(cfg, seed=seed, device=dev)
    enc = V.NativeCLIPVisionEncoder(cfg, sd, dev)
    g = torch.Generator().manual_seed(seed)
    px = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=g).to(dev)
    got = enc.encode(px).float()
    tc = transformers.CLIPVisionConfig(hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                                       num_hidden_layers=cfg.num_hidden_layers,
                                       num_attention_heads=cfg.num_attention_heads, image_size=cfg.image_size,
                                       patch_size=cfg.patch_size, hidden_act=cfg.hidden_act,
                                       projection_dim=cfg.projection_dim, layer_norm_eps=cfg.layer_norm_eps)
    m = transformers.CLIPVisionModelWithProjection(tc).to(dev).eval()
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing)
    with torch.no_grad():
        ref = m(pixel_values=px.half().float()).image_embeds
    err = rel_l2(got, ref)
    print(f"vision tower {cfg.hidden_size}x{cfg.num_hidden_layers} B{B}: image_embeds rel-L2 vs fp32 {err:.3e}")
    enc.close()
    assert torch.isfinite(got).all() and err <= final_tol


def test_vision_tower_tiny():
    """2 layers, heads of 80 padded to 128, 17 tokens; image_embeds within rel-L2 2e-3 of transformers fp32 (the fp16
    activations' rounding)."""
    from cfgpp_b200 import vision_encoder as V
    for B in (1, 3):
        _vision_case(V.tiny_vision_config(), B, 2e-3)


@pytest.mark.parametrize("which", ["vit_h", "vit_bigg"])
def test_vision_tower_production(which):
    """ViT-H/14 (32 layers, heads of 80) and ViT-bigG/14 (48 layers, heads of 104) at 224² (257 tokens), batch 2:
    image_embeds within rel-L2 1e-2 of transformers fp32 on the same fp16 weights (32 / 48 layers of fp16 residual
    stream)."""
    from cfgpp_b200 import vision_encoder as V
    _vision_case(getattr(V, f"{which}_config")(), 2, 1e-2)


@pytest.mark.parametrize("family", ["sd", "sdxl"])
def test_solver_sample_with_ip_adapter(family):
    """sample(ip_adapter=, ip_adapter_image=) end to end on tiny UNets with the tiny tower: fused and callback paths
    give the same image, one image broadcasts like the same image given per prompt, the adapter moves the image, it
    composes with a ControlNet, scale 0 gives the plain image bit for bit, and a later call without it is the plain
    image again. The refiner refuses it."""
    from types import SimpleNamespace
    import numpy as np
    from helpers import rel_l2
    from cfgpp_b200 import config as C, controlnet as CN, ip_adapter as IP, latent_diffusion as LD
    from cfgpp_b200 import latent_sdxl as LX, weights as Wt
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
    img2 = np.ascontiguousarray(img[::-1])
    ad = IP.IPAdapter("ip-solver", dev, cfg)

    def run(**kw):
        if family == "sd":
            s.sample(cfg_guidance=0.6, prompt=["", ["a cat", "a dog"]], zT=zT, **kw)
        else:
            s.sample(prompt1=["", ["a cat", "a dog"]], prompt2=["", ["a cat", "a dog"]], cfg_guidance=0.6,
                     target_size=(8 * hw, 8 * hw), zT=zT, **kw)
        return vae.latents[-1].float()

    plain = run()
    fused = run(ip_adapter=ad, ip_adapter_image=img, ip_adapter_scale=0.8)
    assert rel_l2(fused, plain) >= 1e-2  # deterministic: without the image segment it is `plain` bit for bit
    assert torch.equal(run(ip_adapter=ad, ip_adapter_image=img, ip_adapter_scale=0.8, callback_fn=lambda i, t, kw: kw),
                       fused)
    assert torch.equal(run(ip_adapter=ad, ip_adapter_image=[img, img], ip_adapter_scale=0.8), fused)
    two = run(ip_adapter=ad, ip_adapter_image=[img, img2], ip_adapter_scale=0.8)
    assert torch.equal(two[0], fused[0]) and not torch.equal(two[1], fused[1])
    assert torch.equal(run(ip_adapter=ad, ip_adapter_image=img, ip_adapter_scale=0.0), plain)
    cn = CN.ControlNet("synthetic-controlnet", dev, base_cfg=cfg)
    both = run(ip_adapter=ad, ip_adapter_image=img, ip_adapter_scale=0.8, controlnet=cn,
               control_image=torch.rand(1, 3, 8 * hw, 8 * hw, generator=g))
    assert torch.isfinite(both).all() and rel_l2(both, fused) >= 1e-2
    assert torch.equal(run(), plain) and s.unet.ip_adapter is None
    with pytest.raises(ValueError, match="ip_adapter_image"):
        run(ip_adapter=ad, ip_adapter_image=[img, img, img])
