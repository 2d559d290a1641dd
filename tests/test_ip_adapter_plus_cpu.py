"""IP-Adapter Plus on the host: the Resampler census and its errors, the oracle against an independent fp64
restatement of the original IP-Adapter `Resampler`, the oracle at scale 0, and the unconditional rows."""
import math
import sys
from pathlib import Path

import pytest
import torch

from cfgpp_b200 import config as C, ip_adapter as IP

sys.path.insert(0, str(Path(__file__).resolve().parent))
import ip_adapter_plus_oracle as PO  # noqa: E402

GEOMETRIES = {"sd15": dict(num_queries=16, embed_dim=1280, dim=768, heads=12, depth=4, ff_mult=4),
              "sdxl": dict(num_queries=16, embed_dim=1280, dim=1280, heads=20, depth=4, ff_mult=4)}


@pytest.mark.parametrize("name", ["sd15", "sdxl"])
def test_census_of_the_stated_layout(name):
    """A dict in the released Plus files' layout (image_proj.{latents, proj_in, proj_out, norm_out,
    layers.{i}.{0.norm1, 0.norm2, 0.to_q, 0.to_kv, 0.to_out, 1.0, 1.1, 1.3}}, ip_adapter.{i}.to_{k,v}_ip) is a
    Resampler, and its dimensions are inferred as diffusers does."""
    cfg = C.CONFIGS[name]()
    g = GEOMETRIES[name]
    D = cfg.cross_attention_dim
    shapes = {"image_proj.latents": (1, 16, g["dim"]), "image_proj.proj_in.weight": (g["dim"], 1280),
              "image_proj.proj_in.bias": (g["dim"],), "image_proj.proj_out.weight": (D, g["dim"]),
              "image_proj.proj_out.bias": (D,), "image_proj.norm_out.weight": (D,), "image_proj.norm_out.bias": (D,)}
    for i in range(4):
        l = f"image_proj.layers.{i}."
        shapes.update({l + "0.norm1.weight": (g["dim"],), l + "0.norm1.bias": (g["dim"],),
                       l + "0.norm2.weight": (g["dim"],), l + "0.norm2.bias": (g["dim"],),
                       l + "0.to_q.weight": (64 * g["heads"], g["dim"]),
                       l + "0.to_kv.weight": (128 * g["heads"], g["dim"]),
                       l + "0.to_out.weight": (g["dim"], 64 * g["heads"]), l + "1.0.weight": (g["dim"],),
                       l + "1.0.bias": (g["dim"],), l + "1.1.weight": (4 * g["dim"], g["dim"]),
                       l + "1.3.weight": (g["dim"], 4 * g["dim"])})
    assert IP.resampler_shapes(g, D) == shapes
    sd = {k: torch.zeros(v) for k, v in shapes.items()}
    C_ = IP.block_channels(cfg)
    for i, b in IP.processor_blocks(cfg).items():
        sd[f"ip_adapter.{i}.to_k_ip.weight"] = torch.zeros(C_[b], D)
        sd[f"ip_adapter.{i}.to_v_ip.weight"] = torch.zeros(C_[b], D)
    assert IP.is_resampler(sd) and not IP.is_resampler({**sd, "image_proj.proj.weight": torch.zeros(1)})
    w, geo = IP.resampler_to_unet_keys(sd, cfg)
    assert geo == g
    assert len(w) == len(sd) and all(k in w for k in shapes)
    b1 = IP.processor_blocks(cfg)[1]
    assert w[b1 + ".attn2.processor.to_k_ip.0.weight"] is sd["ip_adapter.1.to_k_ip.weight"]


def test_census_errors():
    cfg = C.CONFIGS["tiny_sd15"]()
    base = IP.synthetic_ip_adapter_plus(cfg, IP.plus_geometry(cfg, 320), seed=1)
    dim = 128

    def err(sd, match):
        with pytest.raises(ValueError, match=match):
            IP.resampler_to_unet_keys(sd, cfg)

    err({**base, "image_proj.pos_emb.weight": torch.zeros(257, 320)}, r"image_proj\.pos_emb\.weight: not a weight")
    err({**base, "image_proj.to_latents_from_mean_pooled_seq.0.weight": torch.zeros(1)},
        r"image_proj\.to_latents_from_mean_pooled_seq\.0\.weight: not a weight")
    err({**base, "image_proj.proj.0.weight": torch.zeros(1280, 320)}, r"image_proj\.proj\.0\.weight: not a weight")
    err({k: v for k, v in base.items() if k != "image_proj.layers.1.0.to_kv.weight"},
        r"image_proj\.layers\.1\.0\.to_kv\.weight: missing")
    err({k: v for k, v in base.items() if k != "image_proj.norm_out.bias"}, r"image_proj\.norm_out\.bias: missing")
    err({**base, "image_proj.layers.0.0.to_q.weight": torch.zeros(100, dim)},
        r"image_proj\.layers\.0\.0\.to_q\.weight: .* 64-wide heads")
    err({**base, "image_proj.layers.1.0.to_kv.weight": torch.zeros(2 * 128 + 64, dim)},
        r"image_proj\.layers\.1\.0\.to_kv\.weight: shape")
    err({**base, "image_proj.latents": torch.zeros(1, 65, dim)}, r"image_proj\.latents: shape")
    err({**base, "image_proj.proj_out.weight": torch.zeros(cfg.cross_attention_dim + 8, dim)},
        r"image_proj\.proj_out\.weight: shape")
    err({**base, "image_proj.layers.1.1.1.weight": torch.zeros(3 * dim, dim)}, r"image_proj\.layers\.1\.1\.1\.weight: shape")
    err({k: v for k, v in base.items() if k != "ip_adapter.31.to_v_ip.weight"}, r"ip_adapter\.31\.to_v_ip\.weight: missing")
    # the plain census still refuses a Resampler key (IPAdapter dispatches on the key set first)
    with pytest.raises(ValueError, match=r"image_proj\.latents: unsupported image projection"):
        IP.to_unet_keys(base, cfg)


def test_plus_adapter_loads_from_file_and_checks_the_encoder(tmp_path):
    from safetensors.torch import save_file
    cfg = C.CONFIGS["tiny_sdxl"]()
    sd = IP.synthetic_ip_adapter_plus(cfg, IP.plus_geometry(cfg, 320), seed=2)
    path = tmp_path / "plus.safetensors"
    save_file(sd, str(path))
    ad = IP.IPAdapter(str(path), "cpu", cfg)
    assert ad.resampler == {**IP.plus_geometry(cfg, 320), "seq_len": 17} and ad.n_tokens == 16
    assert torch.equal(ad.weights["image_proj.latents"], sd["image_proj.latents"])
    syn = IP.IPAdapter("plus-key", "cpu", cfg, image_proj="resampler")
    assert syn.resampler is not None and IP.IPAdapter("plain-key", "cpu", cfg).resampler is None
    bad = {**sd, "image_proj.proj_in.weight": torch.zeros(128, 384)}
    save_file(bad, str(tmp_path / "bad.safetensors"))
    with pytest.raises(ValueError, match=r"image_proj\.proj_in\.weight"):
        IP.IPAdapter(str(tmp_path / "bad.safetensors"), "cpu", cfg)
    with pytest.raises(ValueError, match="image_proj="):
        IP.IPAdapter("k", "cpu", cfg, image_proj="mlp")
    # with a checkpoint, image_proj must name the kind its keys hold
    assert IP.IPAdapter(str(path), "cpu", cfg, image_proj="resampler").resampler is not None
    with pytest.raises(ValueError, match=r"image_proj='linear': .* holds a Resampler"):
        IP.IPAdapter(str(path), "cpu", cfg, image_proj="linear")
    save_file(IP.synthetic_ip_adapter(cfg, 64, seed=3), str(tmp_path / "plain.safetensors"))
    with pytest.raises(ValueError, match=r"image_proj='resampler': .* holds the plain linear projection"):
        IP.IPAdapter(str(tmp_path / "plain.safetensors"), "cpu", cfg, image_proj="resampler")
    big = C.CONFIGS["sd15"]()
    assert IP.plus_encoder_config(big, 1280).hidden_size == 1280
    assert IP.plus_encoder_config(C.CONFIGS["sdxl"](), None).hidden_size == 1280
    with pytest.raises(ValueError, match=r"image_proj\.proj_in\.weight"):
        IP.plus_encoder_config(big, 1024)


def _original_resampler_fp64(w, h, heads, depth):
    """The original IP-Adapter `Resampler` (PerceiverAttention + FeedForward), in fp64: q and k each scaled by
    dim_head^(-1/4), k and v from to_kv(...).chunk(2, -1), norm1 on the image features and norm2 on the latents."""
    w = {k: v.double() for k, v in w.items()}
    p = "image_proj."

    def layer_norm(t, name):
        mu = t.mean(-1, keepdim=True)
        var = ((t - mu) ** 2).mean(-1, keepdim=True)
        return (t - mu) / torch.sqrt(var + 1e-5) * w[name + ".weight"] + w[name + ".bias"]

    def heads_of(t):
        b, l, _ = t.shape
        return t.reshape(b, l, heads, -1).permute(0, 2, 1, 3)

    x = h.double() @ w[p + "proj_in.weight"].T + w[p + "proj_in.bias"]
    lat = w[p + "latents"].expand(h.shape[0], -1, -1)
    for i in range(depth):
        l = f"{p}layers.{i}."
        xn, ln_ = layer_norm(x, l + "0.norm1"), layer_norm(lat, l + "0.norm2")
        q = ln_ @ w[l + "0.to_q.weight"].T
        k, v = (torch.cat((xn, ln_), dim=-2) @ w[l + "0.to_kv.weight"].T).chunk(2, dim=-1)
        q, k, v = heads_of(q), heads_of(k), heads_of(v)
        s = 1 / math.sqrt(math.sqrt(q.shape[-1]))
        att = torch.softmax((q * s) @ (k * s).transpose(-2, -1), dim=-1)
        o = (att @ v).permute(0, 2, 1, 3).reshape(lat.shape[0], lat.shape[1], -1)
        lat = o @ w[l + "0.to_out.weight"].T + lat
        f = layer_norm(lat, l + "1.0") @ w[l + "1.1.weight"].T
        f = 0.5 * f * (1 + torch.erf(f / math.sqrt(2)))
        lat = f @ w[l + "1.3.weight"].T + lat
    return layer_norm(lat @ w[p + "proj_out.weight"].T + w[p + "proj_out.bias"], p + "norm_out")


@pytest.mark.parametrize("name", ["tiny_sd15", "sd15"])
def test_oracle_equals_the_original_resampler(name):
    """The oracle (diffusers' arithmetic) in fp64 equals an fp64 restatement of the original `Resampler`; a swap of k
    and v, or of norm1 and norm2, does not."""
    cfg = C.CONFIGS[name]()
    g = IP.plus_geometry(cfg, 320 if name.startswith("tiny") else 1280)
    if not name.startswith("tiny"):
        g = {**g, "depth": 2}
    sd = IP.synthetic_ip_adapter_plus(cfg, g, seed=5)
    w = {k: v.double() for k, v in sd.items() if k.startswith("image_proj.")}
    h = torch.randn(2, 17 if name.startswith("tiny") else 257, g["embed_dim"], generator=torch.Generator().manual_seed(0),
                    dtype=torch.float64)
    want = _original_resampler_fp64(w, h, g["heads"], g["depth"])
    got = PO.resampler(w, h, g["heads"], g["depth"])
    rel = ((got - want).norm() / want.norm()).item()
    assert rel <= 1e-10, rel
    for a, b in (("0.to_kv.weight", None), ("0.norm1.weight", "0.norm2.weight")):
        bad = dict(w)
        l = "image_proj.layers.0."
        if b is None:
            bad[l + a] = torch.cat(w[l + a].chunk(2, 0)[::-1])
        else:
            bad[l + a], bad[l + b] = w[l + b], w[l + a]
        assert ((PO.resampler(bad, h, g["heads"], g["depth"]) - want).norm() / want.norm()).item() > 1e-3


def test_plus_oracle_at_scale_zero_is_the_plain_oracle():
    import controlnet_oracle as CO
    from oracle import unet as O
    from cfgpp_b200 import weights as Wt
    cfg = C.CONFIGS["tiny_sd15"]()
    sd = Wt.synthetic_state_dict(cfg, seed=7, device="cpu")
    ad = IP.IPAdapter("k", "cpu", cfg, image_proj="resampler")
    g = torch.Generator().manual_seed(0)
    z = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=g)
    t = torch.tensor(301.0)
    m = O.build_unet(CO.oracle_cfg(cfg), sd)
    with torch.no_grad():
        plain = CO.unet_forward(m, z, t, ctx)["sample"]
        st = PO.attach(m, ad.weights, IP.attn2_blocks(cfg), ad.resampler)
        PO.set_hidden_states(st, torch.randn(1, 17, 320, generator=g), torch.randn(1, 17, 320, generator=g))
        assert st["tokens"].shape == (2, 16, cfg.cross_attention_dim)
        st["scale"] = 0.0
        assert torch.equal(CO.unet_forward(m, z, t, ctx)["sample"], plain)
        st["scale"] = 1.0
        assert not torch.allclose(CO.unet_forward(m, z, t, ctx)["sample"], plain)


def test_unconditional_rows_are_the_zero_image_features():
    """IPAdapter hands the native handle the encoder's hidden states of an all-zero preprocessed image as the
    unconditional rows (computed once), not zeros."""
    cfg = C.CONFIGS["tiny_sd15"]()
    ad = IP.IPAdapter("k", "cpu", cfg, image_proj="resampler")
    calls = []

    class Tower:
        def encode_hidden(self, px, skip=1):
            calls.append((px.clone(), skip))
            return torch.full((px.shape[0], 17, 320), 3.0, dtype=torch.float16) + px.flatten(1)[:, :1, None].half()

    ad._encoder = Tower()
    cond = torch.randn(2, 17, 320).half()
    rows = ad.image_rows(cond)
    assert rows.shape == (4, 17, 320)
    assert torch.equal(rows[2:], cond) and torch.all(rows[:2] == 3.0)
    ad.image_rows(cond)
    assert len(calls) == 1 and calls[0][1] == 1 and calls[0][0].shape == (1, 3, 32, 32) and not calls[0][0].any()
