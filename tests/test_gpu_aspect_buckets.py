"""Non-square latents end to end: the SDXL aspect-ratio buckets and the non-square SD v1.5 sizes, whose UNet / VAE
levels the tiled conv A tile cannot address (they take the im2col A tile). Same gates as the square cases:
`test_gpu_unet.run_case` (rel-L2 <= 5e-3 vs the fp16-autocast oracle, fp32 error <= 1.5x the fp16 oracle's own),
`test_gpu_vae._case` / `_enc_case`, and 3e-2 on free-running trajectories like `test_gpu_samplers`.

Latent sizes are (h, w); SDXL's `shape` / `target_size` keep the reference's (W, H) pixel ordering."""
from types import SimpleNamespace

import pytest
import torch

from helpers import build_pair, oracle_cfg, rel_l2
from test_gpu_vae import _case as vae_decode_case, _enc_case as vae_encode_case

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
TOL = 5e-3

# every official SDXL bucket (latent h x w) besides 128 x 128
SDXL_BUCKETS = [(96, 128), (128, 96), (144, 112), (112, 144), (152, 104), (104, 152), (168, 96), (96, 168), (192, 80),
                (80, 192)]


def bucket_inputs(cfg, B, h, w, seed=7):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 4, h, w, generator=g).to(dev)
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    add = None
    if cfg.addition_embed_type == "text_time":
        pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().to(dev)
        tid = torch.tensor([[h * 8, w * 8, 0, 0, h * 8, w * 8]] * (2 * B), dtype=torch.float16).to(dev)
        add = {"text_embeds": pooled, "time_ids": tid}
    return z, uc, c, add


def bind(net, uc, c, add):
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"] if add else None, add["time_ids"].float() if add else None)


def run_case(name, B, h, w, t):
    from oracle import unet as O
    cfg, sd, net, ref16 = build_pair(name, dev)
    z, uc, c, add = bucket_inputs(cfg, B, h, w)
    net.prepare(B, h, w)
    bind(net, uc, c, add)
    eu, ec = net.predict_noise(z, float(t))
    got = torch.cat([eu, ec]).float()
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
    r16 = ref16(z_in, t_in, ctx, add)["sample"].float()
    del ref16
    m32 = O.build_unet(oracle_cfg(cfg), sd, dtype=torch.float32, device=dev)
    with torch.no_grad():
        r32 = m32(z_in, t_in, ctx.float(), {k: v.float() for k, v in add.items()} if add else None)["sample"]
    del m32
    net.close()
    e16, e32, b32 = rel_l2(got, r16), rel_l2(got, r32), rel_l2(r16, r32)
    print(f"{name} B={B} latent {h}x{w}: vs fp16 oracle {e16:.3e}, vs fp32 {e32:.3e} (fp16 oracle itself {b32:.3e})")
    assert got.shape == (2 * B, 4, h, w) and torch.isfinite(got).all()
    assert e16 <= TOL
    assert e32 <= 1.5 * b32 + 1e-4


@pytest.mark.parametrize("name,h,w,t", [("tiny_sdxl", 104, 152, 801), ("tiny_sdxl", 152, 104, 401),
                                        ("tiny_sdxl", 96, 168, 21), ("tiny_sdxl", 80, 192, 981),
                                        ("tiny_sd15", 64, 96, 501), ("tiny_sd15", 96, 64, 301)])
def test_unet_forward_buckets_tiny(name, h, w, t):
    run_case(name, 1, h, w, t)


def test_unet_forward_sdxl_full_size_bucket():
    """The real SDXL UNet at 1216 x 832 px (latent 152 x 104: levels 152x104, 76x52, 38x26)."""
    run_case("sdxl", 1, 152, 104, 501)


def test_unet_forward_sd15_full_size_768x512():
    """The real SD v1.5 UNet at 768 x 512 px (latent 96 x 64; its lowest level is 12 x 8)."""
    run_case("sd15", 1, 96, 64, 401)


def test_bucket_batch2_equals_batch1_per_image():
    cfg, sd, net, _ = build_pair("tiny_sdxl", dev)
    h, w = 104, 152
    z, uc, c, add = bucket_inputs(cfg, 2, h, w)
    net.prepare(2, h, w)
    bind(net, uc, c, add)
    a = net.predict_noise(z, 500.0)
    for i in range(2):
        net.prepare(1, h, w)
        one = {"text_embeds": add["text_embeds"][[i, 2 + i]], "time_ids": add["time_ids"][[i, 2 + i]]}
        bind(net, uc[i:i + 1], c[i:i + 1], one)
        s = net.predict_noise(z[i:i + 1], 500.0)
        e = max(rel_l2(s[0], a[0][i:i + 1]), rel_l2(s[1], a[1][i:i + 1]))
        print(f"bucket {h}x{w}: image {i} batch 1 vs batch 2 rel-L2 {e:.3e}")
        assert e < 1e-3
    net.close()


def test_prepare_accepts_buckets_and_rejects_below_floor():
    from cfgpp_b200 import _native as nv
    cfg, sd, net, _ = build_pair("tiny_sdxl", dev)
    z, uc, c, add = bucket_inputs(cfg, 1, 104, 152)
    net.prepare(1, 104, 152)
    bind(net, uc, c, add)
    a = net.predict_noise(z, 500.0)
    for h, w in SDXL_BUCKETS + [(128, 128)]:
        net.prepare(1, h, w)
    # below the 64 x 64 floor with levels the tiled A tile cannot address (56x40, 40x104, 104x60), or not a multiple
    # of 2^(levels-1) = 4 (66x64)
    for h, w in [(56, 40), (40, 104), (104, 60), (66, 64)]:
        with pytest.raises(nv.NativeError):
            net.prepare(1, h, w)
    net.prepare(1, 104, 152)
    bind(net, uc, c, add)
    b = net.predict_noise(z, 500.0)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    net.close()


# ---- VAE --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,h,w", [(1, 64, 96), (2, 96, 64), (1, 72, 80)])
def test_vae_decode_tiny_non_square(B, h, w):
    vae_decode_case("tiny_vae", B, h, w)


def test_vae_decode_sdxl_bucket():
    """The real decoder at latent 104 x 152 -> 832 x 1216 image (levels up to 832 x 1216, 128-wide row segments
    impossible at every level)."""
    vae_decode_case("sdxl_vae", 1, 104, 152)


def test_vae_encode_sdxl_bucket():
    """A 1216 x 832 image through the real encoder (stride-2 pad-after convs at 1216x832 -> 152x104)."""
    vae_encode_case("sdxl_vae", 1, 1216, 832, check32=False)


# ---- trajectories -----------------------------------------------------------------------------------------------
def test_bucket_ddim_and_dpmpp_trajectories_vs_oracle():
    from cfgpp_b200 import schedule as S
    from oracle import samplers as OSm, schedule as OS
    cfg, sd, net, ref = build_pair("tiny_sdxl", dev)
    h, w, nfe, lam = 104, 152, 6, 0.6
    z, uc, c, add = bucket_inputs(cfg, 1, h, w)
    tb = OS.make_tables(nfe)
    sch = S.Schedule.make(nfe)
    net.prepare(1, h, w)
    bind(net, uc, c, add)
    z0_ref = OSm.sdxl_ddim_cfgpp(ref, tb, z, uc, c, lam, add)
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, S.ddim_cfgpp_steps(sch, lam, True))
    net.set_state(z)
    net.run_steps(0, nfe)
    e = rel_l2(net.get_state(1), z0_ref)
    print(f"tiny_sdxl {h}x{w} ddim_cfg++ NFE={nfe}: rel-L2 final z0t {e:.3e}")
    assert e <= 3e-2
    x_ref = OSm.sdxl_dpmpp_2m_cfgpp(ref, tb, z, uc, c, lam, add)
    steps, sigma0 = S.dpmpp_2m_cfgpp_steps(sch, lam)
    net.set_schedule(S.STEP_DPMPP2M_CFGPP, torch.float16, steps)
    net.set_state(z.to(torch.float16) * sigma0)
    net.run_steps(0, len(steps))
    e = rel_l2(net.get_state(0), x_ref)
    print(f"tiny_sdxl {h}x{w} dpm++_2m_cfgpp NFE={nfe}: rel-L2 final x {e:.3e}")
    assert e <= 3e-2
    net.close()


def test_bucket_fused_equals_callback_path():
    from cfgpp_b200 import schedule as S
    cfg, sd, net, _ = build_pair("tiny_sdxl", dev)
    h, w = 152, 104
    z, uc, c, add = bucket_inputs(cfg, 2, h, w)
    steps = S.ddim_cfgpp_steps(S.Schedule.make(5), 0.6, True)
    net.prepare(2, h, w)
    bind(net, uc, c, add)
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
    net.set_state(z)
    net.run_steps(0, len(steps))
    a0, a1 = net.get_state(0).clone(), net.get_state(1).clone()
    net.set_state(z)
    for i, st in enumerate(steps):
        eu, ec = net.predict_noise(net.get_state(0), st.t)
        net.apply_step(i, eu, ec)
    assert torch.equal(a0, net.get_state(0)) and torch.equal(a1, net.get_state(1))
    net.close()


def test_sdxl_sample_at_bucket_target_size():
    """`sample(target_size=(832, 1216))` — (W, H) as in the reference — returns a 1216 x 832 image, equal to decoding
    `reverse_process` on the same seeded zT by hand."""
    from cfgpp_b200 import latent_sdxl as LX
    from cfgpp_b200.config import tiny_sdxl_config
    from cfgpp_b200.utils.log_util import set_seed
    s = LX.get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=3), device="cuda:0",
                      unet_config=tiny_sdxl_config(), model_key="synthetic:7")
    set_seed(42)
    img = s.sample(prompt1=["", "a cat"], prompt2=["", "a cat"], cfg_guidance=0.6, original_size=(832, 1216),
                   target_size=(832, 1216))
    assert img.shape == (1, 3, 1216, 832) and torch.isfinite(img).all() and 0 <= img.min() and img.max() <= 1
    set_seed(42)
    uc, c, pn, pc = s.get_text_embed("", "a cat", "", "a cat")
    tid = torch.tensor([[832., 1216, 0, 0, 832, 1216]] * 2).half().to(dev)
    add = {"text_embeds": torch.cat([pn, pc]).to(dev), "time_ids": tid}
    z0 = s.reverse_process(uc, c, 0.6, add, (832, 1216))
    assert z0.shape == (1, 4, 152, 104)
    by_hand = (s.decode(z0) / 2 + 0.5).clamp(0, 1).cpu()
    assert torch.equal(img, by_hand)
    LX.release_engines()


def test_sd15_sample_with_non_square_zT():
    from cfgpp_b200 import latent_diffusion as LD
    from cfgpp_b200.config import tiny_sd15_config
    s = LD.get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=3), device="cuda:0",
                      unet_config=tiny_sd15_config(), model_key="synthetic:9")
    g = torch.Generator().manual_seed(3)
    zT = torch.randn(1, 4, 96, 64, generator=g)
    img = s.sample(prompt=["", "a dog"], cfg_guidance=0.6, zT=zT)
    assert img.shape == (1, 3, 768, 512) and torch.isfinite(img).all()
    again = s.sample(prompt=["", "a dog"], cfg_guidance=0.6, zT=zT)
    assert torch.equal(img, again)
