"""UNet forward parity through the C ABI against the oracle on the same seeded weights / inputs.

Stated tolerance (BASELINE.md §3, SURVEY §8c): rel-L2(eps_native, eps_ref16) <= 5e-3 where ref16 is the restated
UNet under torch.autocast('cuda', fp16) (the reference's op sequence), AND the error against the fp32 oracle must
not exceed 1.5x the fp16 reference's own error. Both errors are printed by the tests."""
import pytest
import torch

from helpers import build_pair, make_inputs, oracle_cfg, rel_l2

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
TOL = 5e-3


def run_case(name, B, hw, t, dup=True):
    from oracle import unet as O
    cfg, sd, net, ref16 = build_pair(name, dev)
    z, uc, c, add = make_inputs(cfg, B, hw, dev, duplicate_added=dup)
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"] if add else None, add["time_ids"].float() if add else None)
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
    assert torch.isfinite(got).all()
    assert rel_l2(got, r16) <= TOL
    assert rel_l2(got, r32) <= 1.5 * rel_l2(r16, r32) + 1e-4
    return got, r16


@pytest.mark.parametrize("name,B,hw,t", [("tiny_sdxl", 2, 32, 801), ("tiny_sd15", 1, 32, 401), ("tiny_sdxl", 1, 64, 21),
                                         ("tiny_sd15", 4, 16, 981)])
def test_unet_forward_tiny(name, B, hw, t):
    run_case(name, B, hw, t)


def test_unet_forward_lightning_style_undup_added_cond():
    """cfg_guidance == 1: the reference passes un-duplicated added conditions which diffusers broadcasts over the
    batch of 2 (latent_sdxl.py:249-252; SURVEY Appendix C.8)."""
    run_case("tiny_sdxl", 1, 32, 999, dup=False)


def test_unet_forward_landscape_latent():
    """A 4:3 aspect bucket (latent 96 x 128 = 768 x 1024 px): power-of-two width, H a multiple of the rows per conv
    tile at every level (96x128, 48x64, 24x32) — the reference takes any `shape` (latent_sdxl.py:720)."""
    from oracle import unet as O
    cfg, sd, net, ref16 = build_pair("tiny_sdxl", dev)
    g = torch.Generator().manual_seed(3)
    B, h, w = 1, 96, 128
    z = torch.randn(B, 4, h, w, generator=g).to(dev)
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    add = {"text_embeds": torch.randn(2 * B, cfg.pooled_dim, generator=g).half().to(dev),
           "time_ids": torch.tensor([[768., 1024, 0, 0, 768, 1024]] * (2 * B)).half().to(dev)}
    net.prepare(B, h, w)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
    eu, ec = net.predict_noise(z, 333.0)
    got = torch.cat([eu, ec]).float()
    r16 = ref16(torch.cat([z] * 2), torch.tensor(333, device=dev), torch.cat([uc, c]), add)["sample"].float()
    e = rel_l2(got, r16)
    print(f"tiny_sdxl 96x128 latent: rel-L2 vs fp16 oracle {e:.3e}")
    assert got.shape == (2, 4, 96, 128) and e <= TOL
    net.close()


def test_unet_forward_sdxl_full_size():
    """BASELINE config 3 geometry: SDXL, 128x128 latent (1024^2), UNet batch 2 (one image, uncond+cond)."""
    run_case("sdxl", 1, 128, 501)


def test_unet_forward_sd15_full_size():
    """BASELINE configs[0]/[1] geometry: the real SD v1.5 UNet (859.5 M params, head dims 40/80/160, 1x1-conv
    projections, 8x8 deepest level), 64x64 latent."""
    run_case("sd15", 1, 64, 401)


def test_forward_is_deterministic_and_rows_independent():
    cfg, sd, net, _ = build_pair("tiny_sdxl", dev)
    z, uc, c, add = make_inputs(cfg, 2, 32, dev)
    net.prepare(2, 32, 32)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
    a = net.predict_noise(z, 500.0)
    b = net.predict_noise(z, 500.0)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])  # idempotent, no atomics on the data path
    # image 0 alone (batch 1) gives the same eps as image 0 inside the batch of 2
    net.prepare(1, 32, 32)
    net.set_prompt(torch.cat([uc[:1], c[:1]]), add["text_embeds"][[0, 2]], add["time_ids"][[0, 2]].float())
    s = net.predict_noise(z[:1], 500.0)
    assert rel_l2(s[0], a[0][:1]) < 1e-3 and rel_l2(s[1], a[1][:1]) < 1e-3
    net.close()


@pytest.mark.parametrize("name", ["tiny_sdxl", "tiny_sd15"])
def test_native_unet_against_committed_golden(name):
    """Native forward vs the COMMITTED fp32-oracle vectors (tests/golden/r01_golden.pt): same seeded CPU weights, same
    inputs; stated tolerance rel-L2 <= 5e-3 (fp16 path against an fp32 result)."""
    from pathlib import Path
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    gold = torch.load(Path(__file__).parent / "golden" / "r01_golden.pt", weights_only=False)["unet"][name]
    cfg = C.CONFIGS[name]()
    sd = {k: v.to(dev) for k, v in Wt.synthetic_state_dict(cfg, seed=gold["seed"], device="cpu").items()}
    net = NativeUNet(cfg, sd, dev)
    hw = gold["hw"]
    net.prepare(1, hw, hw)
    add = gold["add"]
    net.set_prompt(gold["ctx"].to(dev), None if add is None else add["text_embeds"].to(dev),
                   None if add is None else add["time_ids"].float().to(dev))
    eu, ec = net.predict_noise(gold["z"].to(dev), float(gold["t"]))
    e_uc, e_c = rel_l2(eu.cpu(), gold["eps_uc"]), rel_l2(ec.cpu(), gold["eps_c"])
    print(f"{name} vs golden fp32: rel-L2 eps_uc {e_uc:.3e} eps_c {e_c:.3e}")
    assert e_uc <= 5e-3 and e_c <= 5e-3
    net.close()
