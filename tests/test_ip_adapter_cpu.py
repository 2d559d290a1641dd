"""IP-Adapter on the host: the processor-index mapping, the checkpoint loaders and their errors, and the oracle's
adapter at scale 0."""
import pytest
import torch

from cfgpp_b200 import config as C, ip_adapter as IP


def test_processor_index_mapping_production():
    """diffusers counts attn1 and attn2 of every transformer block in attn_processors order (down, up, mid): attn2 at
    the odd indices, the mid block last."""
    sd15 = IP.processor_blocks(C.CONFIGS["sd15"]())
    assert sorted(sd15) == list(range(1, 32, 2))
    assert sd15[1] == "down_blocks.0.attentions.0.transformer_blocks.0"
    assert sd15[11] == "down_blocks.2.attentions.1.transformer_blocks.0"
    assert sd15[13] == "up_blocks.1.attentions.0.transformer_blocks.0"
    assert sd15[29] == "up_blocks.3.attentions.2.transformer_blocks.0"
    assert sd15[31] == "mid_block.attentions.0.transformer_blocks.0"
    sdxl = IP.processor_blocks(C.CONFIGS["sdxl"]())
    assert sorted(sdxl) == list(range(1, 140, 2))
    assert sdxl[1] == "down_blocks.1.attentions.0.transformer_blocks.0"
    assert sdxl[47] == "down_blocks.2.attentions.1.transformer_blocks.9"
    assert sdxl[49] == "up_blocks.0.attentions.0.transformer_blocks.0"
    assert sdxl[119] == "up_blocks.1.attentions.2.transformer_blocks.1"
    assert sdxl[121] == "mid_block.attentions.0.transformer_blocks.0"
    assert sdxl[139] == "mid_block.attentions.0.transformer_blocks.9"
    ch = IP.block_channels(C.CONFIGS["sdxl"]())
    assert ch[sdxl[1]] == 640 and ch[sdxl[49]] == 1280 and ch[sdxl[119]] == 640 and ch[sdxl[139]] == 1280


@pytest.mark.parametrize("name,n", [("tiny_sd15", 16), ("tiny_sdxl", 17)])
def test_processor_index_mapping_tiny(name, n):
    cfg = C.CONFIGS[name]()
    blocks = IP.processor_blocks(cfg)
    assert sorted(blocks) == list(range(1, 2 * n, 2))
    assert blocks[2 * n - 1].startswith("mid_block.")
    assert [b.split(".")[0] for b in blocks.values()] == sorted(
        (b.split(".")[0] for b in blocks.values()), key=["down_blocks", "up_blocks", "mid_block"].index)


def _sd(cfg):
    return IP.synthetic_ip_adapter(cfg, embed_dim=64, n_tokens=4, seed=3)


@pytest.mark.parametrize("fmt", [".bin", ".safetensors"])
def test_loader_round_trip(tmp_path, fmt):
    cfg = C.CONFIGS["tiny_sdxl"]()
    sd = _sd(cfg)
    path = tmp_path / f"ip{fmt}"
    if fmt == ".bin":
        nested = {top: {k[len(top) + 1:]: v for k, v in sd.items() if k.startswith(top + ".")}
                  for top in ("image_proj", "ip_adapter")}
        torch.save(nested, path)
    else:
        from safetensors.torch import save_file
        save_file(sd, str(path))
    ad = IP.IPAdapter(str(path), "cpu", cfg)
    assert (ad.n_tokens, ad.embed_dim) == (4, 64)
    blocks = IP.processor_blocks(cfg)
    for i, b in blocks.items():
        assert torch.equal(ad.weights[b + ".attn2.processor.to_k_ip.0.weight"], sd[f"ip_adapter.{i}.to_k_ip.weight"])
        assert torch.equal(ad.weights[b + ".attn2.processor.to_v_ip.0.weight"], sd[f"ip_adapter.{i}.to_v_ip.weight"])
    assert torch.equal(ad.weights["image_proj.proj.weight"], sd["image_proj.proj.weight"])
    assert len(ad.weights) == 4 + 2 * len(blocks)


def test_synthetic_key_is_seeded():
    cfg = C.CONFIGS["tiny_sd15"]()
    a, b = IP.IPAdapter("some-adapter", "cpu", cfg), IP.IPAdapter("some-adapter", "cpu", cfg)
    assert all(torch.equal(a.weights[k], b.weights[k]) for k in a.weights)
    assert not torch.equal(IP.IPAdapter("other", "cpu", cfg).weights["image_proj.proj.weight"],
                           a.weights["image_proj.proj.weight"])


def test_loader_errors(tmp_path):
    cfg = C.CONFIGS["tiny_sd15"]()
    D = cfg.cross_attention_dim

    def err(sd, match):
        with pytest.raises(ValueError, match=match):
            IP.to_unet_keys(sd, cfg)

    base = _sd(cfg)
    err({**base, "ip_adapter.1.to_q_ip.weight": torch.zeros(1)}, r"ip_adapter\.1\.to_q_ip\.weight: not an IP-Adapter")
    err({**base, "image_proj.latents": torch.zeros(1, 16, D)}, r"image_proj\.latents: unsupported image projection")
    err({**base, "ip_adapter.33.to_k_ip.weight": torch.zeros(64, D)}, r"ip_adapter\.33\.to_k_ip\.weight: processor")
    err({**base, "ip_adapter.2.to_k_ip.weight": torch.zeros(64, D)}, r"ip_adapter\.2\.to_k_ip\.weight: processor")
    err({k: v for k, v in base.items() if k != "ip_adapter.31.to_v_ip.weight"}, r"ip_adapter\.31\.to_v_ip\.weight: missing")
    err({**base, "ip_adapter.1.to_k_ip.weight": torch.zeros(128, D)}, r"ip_adapter\.1\.to_k_ip\.weight: shape")
    err({**base, "image_proj.norm.weight": torch.zeros(D + 1)}, r"image_proj\.norm\.weight: shape")
    err({**base, "image_proj.proj.weight": torch.zeros(4 * D + 1, 64)}, r"image_proj\.proj\.weight: shape")
    err({k: v for k, v in base.items() if k != "image_proj.norm.bias"}, r"image_proj\.norm\.bias: missing")
    bad = tmp_path / "bad.bin"
    torch.save({"image_proj": {}}, bad)
    with pytest.raises(ValueError, match="image_proj' and 'ip_adapter"):
        IP.IPAdapter(str(bad), "cpu", cfg)
    with pytest.raises(FileNotFoundError, match="does not exist"):
        IP.IPAdapter(str(tmp_path / "missing.safetensors"), "cpu", cfg)
    with pytest.raises(ValueError, match="SD v1.5 and SDXL"):
        IP.IPAdapter("k", "cpu", C.CONFIGS["tiny_sd2"]())


def test_oracle_adapter_at_scale_zero_is_the_plain_oracle():
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent))
    import controlnet_oracle as CO
    import ip_adapter_oracle as IO
    from oracle import unet as O
    from cfgpp_b200 import weights as Wt
    cfg = C.CONFIGS["tiny_sd15"]()
    sd = Wt.synthetic_state_dict(cfg, seed=7, device="cpu")
    ad = IP.IPAdapter("k", "cpu", cfg)
    g = torch.Generator().manual_seed(0)
    z = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=g)
    t = torch.tensor(301.0)
    m = O.build_unet(CO.oracle_cfg(cfg), sd)
    with torch.no_grad():
        plain = CO.unet_forward(m, z, t, ctx)["sample"]
        st = IO.attach(m, ad.weights, IP.attn2_blocks(cfg), ad.n_tokens, cfg.cross_attention_dim)
        IO.set_embeds(st, torch.randn(1, 64, generator=g))
        st["scale"] = 0.0
        assert torch.equal(CO.unet_forward(m, z, t, ctx)["sample"], plain)
        st["scale"] = 1.0
        assert not torch.allclose(CO.unet_forward(m, z, t, ctx)["sample"], plain)


def test_preprocessing_matches_clip_image_processor():
    """Shortest side to 224 (bicubic), center crop, 1/255, CLIP mean / std: equal to transformers' CLIPImageProcessor
    (PIL path) on images of several aspect ratios."""
    transformers = pytest.importorskip("transformers")
    import numpy as np
    from cfgpp_b200 import vision_encoder as V
    cls = getattr(transformers, "CLIPImageProcessorPil", None) or transformers.CLIPImageProcessor  # the PIL path
    proc = cls(size={"shortest_edge": 224}, crop_size={"height": 224, "width": 224})
    g = np.random.default_rng(0)
    for h, w in ((224, 224), (300, 200), (120, 517), (640, 480), (97, 97)):
        img = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        want = proc(images=img, return_tensors="pt")["pixel_values"]
        got = V.preprocess([img])
        assert got.shape == want.shape == (1, 3, 224, 224)
        assert torch.allclose(got, want, atol=1e-6, rtol=0), f"{h}x{w}: max |diff| {(got - want).abs().max()}"


def test_solver_refusals():
    """The inversion / edit solvers (refuse_control) and refiner= (refuse_ip_adapter) refuse an IP-Adapter;
    ip_adapter and ip_adapter_image go together."""
    from cfgpp_b200 import solver_base as SB
    for kw in ({"ip_adapter": object()}, {"ip_adapter_image": object()}):
        with pytest.raises(ValueError, match="does not take an IP-Adapter"):
            SB.refuse_control(kw, "ddim_inversion")
        with pytest.raises(ValueError, match="does not take an IP-Adapter"):
            SB.refuse_ip_adapter(kw, "sample(refiner=...)")
        with pytest.raises(ValueError, match="go together"):
            SB.ip_request(kw, 2)
    assert SB.ip_request({}, 2) is None
    SB.refuse_control({}, "ddim_edit")
