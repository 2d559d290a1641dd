"""The production size table (`production.py`) and the per-element case lists derived from it, checked without a GPU:
every full-size UNet config, text tower, vision tower, ControlNet-capable UNet, IP-Adapter (plain and Plus) and
T2I-capable UNet has sizes, and the GEMM / conv, attention, GroupNorm and LayerNorm case lists cover every (model, size). A model added to `config.CONFIGS` or `text_encoder.CLIP_CONFIGS` without sizes fails here,
on any machine, before its kernels go unpinned."""
import pytest

import production as P
import test_gpu_attention as TA
import test_gpu_gemm as TG
import test_gpu_norms as TN
from cfgpp_b200 import config as C
from cfgpp_b200.text_encoder import CLIP_CONFIGS

# the sizes the pins must keep: each model's native resolution and the non-square sizes whose levels end in partial
# tiles (removing one of these from the table fails here)
REQUIRED_UNET = {"sdxl": {(128, 128), (152, 104)}, "sd15": {(64, 64)}, "sd2": {(96, 96), (96, 64)},
                 "sd2_base": {(64, 64)}, "sdxl_refiner": {(128, 128), (152, 104), (168, 96)}}
REQUIRED_VAE = {(1024, 1024), (1216, 832), (768, 768), (768, 512), (512, 512)}


def full_size(names):
    return sorted(n for n in names if not n.startswith("tiny"))


def test_every_unet_config_has_sizes():
    missing = [m for m in full_size(C.CONFIGS) if not P.UNET_SIZES.get(m)]
    assert not missing, f"full-size UNet configs without production sizes: {missing}"
    for m, sizes in P.UNET_SIZES.items():
        cfg = C.CONFIGS[m]()
        assert (cfg.sample_size, cfg.sample_size) in sizes, f"{m}: its native {cfg.sample_size}² latent is not listed"
        down = 1 << (len(cfg.block_out_channels) - 1)
        for h, w in sizes:
            assert h % down == 0 and w % down == 0, f"{m}: latent {h}x{w} is not a multiple of {down}"


def test_required_sizes_listed():
    for m, sizes in REQUIRED_UNET.items():
        assert sizes <= set(P.UNET_SIZES.get(m, ())), f"{m}: {sorted(sizes - set(P.UNET_SIZES.get(m, ())))} removed"
    assert REQUIRED_VAE <= set(P.VAE_SIZES), f"VAE sizes removed: {sorted(REQUIRED_VAE - set(P.VAE_SIZES))}"


def test_every_text_tower_listed():
    missing = [t for t in full_size(CLIP_CONFIGS) if not P.TEXT_TOWERS.get(t)]
    assert not missing, f"text towers without prompt batches: {missing}"


def expected_keys(vae=True, towers=True):
    keys = {(m, (h, w)) for m, h, w in P.unet_sizes()}
    if vae:
        keys |= {("vae", hw) for hw in P.VAE_SIZES}
    if towers:
        keys |= {(t, B) for t, batches in P.TEXT_TOWERS.items() for B in batches}
    return keys


def assert_covered(what, lists, run, key_of):
    """Every list is non-empty and every entry of it runs (possibly under another model's id, when shared)."""
    for k, entries in lists.items():
        assert entries, f"{what}: no cases derived for {k}"
        lost = [e for e in entries if key_of(e) not in run]
        assert not lost, f"{what}: {len(lost)} launches of {k} do not run, first {lost[0]}"


def test_gemm_cases_cover_every_model_and_size():
    lists = TG.production_lists()
    lists = {k: v for k, v in lists.items()
             if k[0] not in ("controlnet", "ip_adapter", "ip_adapter_plus", "t2i_adapter") and k[0] not in P.VISION_TOWERS}
    assert set(lists) == expected_keys()
    run = {TG.signature(p.values[0]) for p in TG._production_cases()}
    assert_covered("GEMM", lists, run, lambda e: TG.signature(e[1]))


def test_attention_cases_cover_every_model_and_size():
    lists = TA.production_lists()
    assert set(lists) == expected_keys(vae=False, towers=False)
    for k, shapes in lists.items():  # self- and cross-attention at every size
        assert {s[1] == s[2] for _, s in shapes} == {True, False}, f"attention {k}: {shapes}"
    run = {tuple(p.values) for p in TA._production_cases()}
    assert_covered("attention", lists, run, lambda e: e[1])


def test_groupnorm_cases_cover_every_model_and_size():
    lists = TN.production_lists()
    assert set(lists) == expected_keys(towers=False)
    unet = {tuple(c[3:]) for c in TN._unet_cases()}
    vae = {(c[0], *c[3:]) for c in TN._vae_cases()}
    assert_covered("GroupNorm", {k: v for k, v in lists.items() if k[0] != "vae"}, unet, tuple)
    assert_covered("GroupNorm", {k: v for k, v in lists.items() if k[0] == "vae"}, vae, tuple)


@pytest.mark.parametrize("model", sorted(REQUIRED_UNET))
def test_new_levels_reach_the_lists(model):
    """Spot checks of what each model brings: SD 2's 9216-token level at 768², the refiner's 12..96 channels per
    group with concat groups across the source boundary and its 3072-channel conv (K = 27648), SDXL's 3952-token
    level at 1216x832."""
    cfg = C.CONFIGS[model]()
    native = (model, (cfg.sample_size, cfg.sample_size))
    gemm = [l for _, l in TG.production_lists()[native]]
    attn = [s for _, s in TA.production_lists()[native]]
    gn = TN.production_lists()[native]
    ch = cfg.block_out_channels
    assert max(l.get("Cin", 0) for l in gemm) == 2 * ch[-1]
    assert (cfg.num_attention_heads[-1], 77) in {(s[0], s[2]) for s in attn}
    assert {(c1 + c2) // 32 for c1, c2, *_ in gn} >= {c // 32 for c in ch}
    if model == "sdxl_refiner":
        assert {(c1 + c2) // 32 for c1, c2, *_ in gn} >= {12, 24, 36, 48, 72, 96}
        assert (1536, 768) in {(c1, c2) for c1, c2, *_ in gn} and (768, 384) in {(c1, c2) for c1, c2, *_ in gn}
    if model == "sd2":
        assert (5, 9216, 9216, 64) in attn
    if model in ("sdxl", "sdxl_refiner"):
        tall = [s for _, s in TA.production_lists()[(model, (152, 104))]]
        assert any(s[1] == 3952 for s in tall)


# ------------------------------------------------------------------------------------------------ ControlNet, IP-Adapter, vision towers

REQUIRED_CONTROL_BATCHES = {1, 8}
REQUIRED_IP = {("sd15", 1024), ("sdxl", 1280), ("sdxl", 1024)}
NO_CONTROLNET = {"sdxl_refiner"}  # the refiner refuses a ControlNet


def test_every_vision_tower_listed():
    from cfgpp_b200 import vision_encoder as V
    towers = {n[:-len("_config")] for n in dir(V) if n.endswith("_config") and callable(getattr(V, n))}
    missing = [t for t in full_size(towers) if not P.VISION_TOWERS.get(t)]
    assert not missing, f"vision towers without image batches: {missing}"
    for t, batches in P.VISION_TOWERS.items():
        assert {1, 2, 8} <= set(batches), f"{t}: image batches {batches}"


def test_every_controlnet_unet_has_sizes():
    capable = [m for m in full_size(C.CONFIGS) if m not in NO_CONTROLNET]
    for m in capable:
        assert set(P.CONTROLNET_SIZES.get(m, ())) == set(P.UNET_SIZES[m]), f"{m}: ControlNet sizes differ from its sizes"
    assert not NO_CONTROLNET & set(P.CONTROLNET_SIZES), "the refiner takes no ControlNet"
    assert set(P.CONTROLNET_SIZES) == set(capable)
    assert REQUIRED_CONTROL_BATCHES <= set(P.CONTROL_IMAGE_BATCHES)


def test_every_ip_adapter_listed():
    assert REQUIRED_IP <= set(P.IP_ADAPTERS) and P.IP_TOKENS == 4


def test_controlnet_and_vision_gemm_lists_run():
    lists = TG.production_lists()
    want = {("controlnet", m, (h, w)) for m, h, w in P.controlnet_sizes()}
    want |= {(t, B) for t, batches in P.VISION_TOWERS.items() for B in batches}
    want |= {("ip_adapter", m, E) for m, E in P.IP_ADAPTERS}
    assert want <= set(lists)
    run = {TG.signature(p.values[0]) for p in TG._production_cases()}
    assert_covered("GEMM", {k: lists[k] for k in want}, run, lambda e: TG.signature(e[1]))
    kinds = {l.get("addend") for k in want if k[0] == "controlnet" for _, l in lists[k]}
    assert "scaled_residual" in kinds


@pytest.mark.parametrize("model", sorted(P.CONTROLNET_SIZES))
def test_conditioning_embedding_launches_match_param_specs(model):
    """One padded conv per `controlnet_cond_embedding.*` weight, with its Cin, Cout and stride (2 on blocks.1 / 3 / 5)."""
    from cfgpp_b200 import controlnet as CN
    cn_cfg = CN.controlnet_config(C.CONFIGS[model]())
    specs = {k[:-len(".weight")]: shape for k, shape, _ in CN.controlnet_param_specs(cn_cfg)
             if k.startswith("controlnet_cond_embedding.") and k.endswith(".weight")}
    for h, w in P.CONTROLNET_SIZES[model]:
        for B in P.CONTROL_IMAGE_BATCHES:
            got = {l["name"]: l for l in TG.controlnet_embed_launches(cn_cfg, h, w, B)}
            assert set(got) == set(specs)
            for name, (cout, cin, kh, kw) in specs.items():
                l = got[name]
                assert (l["cin_real"], l["cout_real"], kh, kw) == (cin, cout, 3, 3), name
                assert l["Cin"] == TG.pad64(cin) and l["Cout"] >= cout and l["Cout"] % 64 == 0 and l["B"] == B
                assert l["stride"] == (2 if name.endswith(("blocks.1", "blocks.3", "blocks.5")) else 1), name
            assert got["controlnet_cond_embedding.conv_in"]["H"] == 8 * h
        zc = TG.zero_conv_launches(cn_cfg, h, w)
        zspec = {k[:-len(".weight")]: s for k, s, _ in CN.controlnet_param_specs(cn_cfg)
                 if k.startswith(("controlnet_down_blocks.", "controlnet_mid_block")) and k.endswith(".weight")}
        assert {l["name"]: (l["N"], l["K"]) for l in zc} == {k: s[:2] for k, s in zspec.items()}


@pytest.mark.parametrize("model,E", sorted(REQUIRED_IP))
def test_to_kv_ip_launches_match_adapter_keys(model, E):
    """The derived to_kv_ip launches are one per cross-attention block, with K = D and N = 2·Cp for the block's width C
    (the rows of its to_k_ip weight); image_proj.proj takes the E-wide embedding to IP_TOKENS tokens."""
    from cfgpp_b200 import ip_adapter as IP
    cfg = C.CONFIGS[model]()
    sd = IP.synthetic_ip_adapter(cfg, E, P.IP_TOKENS)
    blocks = IP.processor_blocks(cfg)
    launches = TG.ip_adapter_gemm_launches(cfg, E, P.IP_TOKENS)
    proj, kv = launches[0], launches[1:]
    assert (proj["name"], proj["N"], proj["K"]) == ("image_proj.proj", tuple(sd["image_proj.proj.weight"].shape)[0], E)
    want = {blocks[i]: sd[f"ip_adapter.{i}.to_k_ip.weight"].shape for i in blocks}
    got = {l["name"][:-len(".attn2.to_kv_ip")]: l for l in kv}
    assert set(got) == set(want)
    for b, (Cb, D) in want.items():
        H, hd = got[b]["ip_heads"]
        assert H * hd == Cb and got[b]["K"] == D == cfg.cross_attention_dim and got[b]["N"] == 2 * H * TG.pad64(hd)


def test_layernorm_cases_cover_every_tower_and_adapter():
    lists = TN.layernorm_production_lists()
    want = {(t, B) for t, batches in P.TEXT_TOWERS.items() for B in batches}
    want |= {(t, B) for t, batches in P.VISION_TOWERS.items() for B in batches}
    want |= {("ip_adapter", m, E) for m, E in P.IP_ADAPTERS}
    assert set(lists) == want
    run = {tuple(c.values[:2]) for c in TN._layernorm_cases()}
    assert_covered("LayerNorm", lists, run, lambda e: e[1])
    widths = {c for v in lists.values() for _, (M, c) in v}
    assert {768, 1280, 1024, 1664, 2048} <= widths


def test_vision_attention_cases_listed():
    lists = TA.vision_production_lists()
    assert set(lists) == {(t, B) for t, batches in P.VISION_TOWERS.items() for B in batches}
    run = {tuple(p.values) for p in TA._vision_cases()}
    assert_covered("vision attention", lists, run, lambda e: e[1])
    assert {s[3] for v in lists.values() for _, s in v} == {80, 104}


# ------------------------------------------------------------------------------------------------ IP-Adapter Plus, T2I-Adapter

REQUIRED_IP_PLUS = {("sd15", 1280), ("sdxl", 1280)}
# the refiner runs the steps after an SDXL hand-off without the base's T2I features, and no released adapter targets it
NO_T2I = {"sdxl_refiner"}
# adapter sizes beyond the UNet's own: SD v1.5 at 512x768, whose adapter levels are 96/48/24/12 wide (the im2col A tile)
T2I_EXTRA_SIZES = {"sd15": {(64, 96)}}


def test_every_ip_plus_adapter_listed():
    assert REQUIRED_IP_PLUS <= set(P.IP_PLUS_ADAPTERS)
    assert {2, 4, 16} <= set(P.IP_PLUS_NB)


def test_every_t2i_unet_has_sizes():
    capable = [m for m in full_size(C.CONFIGS) if m not in NO_T2I]
    assert set(P.T2I_ADAPTER_SIZES) == set(capable), "T2I-Adapter sizes are not listed for exactly the capable UNets"
    for m in capable:
        want = set(P.UNET_SIZES[m]) | T2I_EXTRA_SIZES.get(m, set())
        assert set(P.T2I_ADAPTER_SIZES[m]) == want, f"{m}: T2I-Adapter sizes {P.T2I_ADAPTER_SIZES[m]}, want {want}"
    assert set(P.T2I_ADAPTER_BATCHES) == {1, 8} and set(P.T2I_IN_CHANNELS) == {1, 3}


def test_adapter_gemm_lists_run():
    lists = TG.production_lists()
    want = {("t2i_adapter", m, (h, w)) for m, h, w in P.t2i_sizes()}
    want |= {("ip_adapter_plus", m, E) for m, E in P.IP_PLUS_ADAPTERS}
    assert want <= set(lists)
    run = {TG.signature(p.values[0]) for p in TG._production_cases()}
    assert_covered("GEMM", {k: lists[k] for k in want}, run, lambda e: TG.signature(e[1]))


@pytest.mark.parametrize("in_channels", P.T2I_IN_CHANNELS)
@pytest.mark.parametrize("model", sorted(P.T2I_ADAPTER_SIZES))
def test_t2i_launches_match_param_specs(model, in_channels):
    """Every `adapter.*` weight of `t2i_adapter_param_specs` is the weight of exactly one derived launch, by name, with
    its (N, K) (a 3x3 conv's K = 9·Cin), and every launch has a weight; block2 adds its residual in place."""
    from cfgpp_b200 import t2i_adapter as T
    cfg = T.t2i_adapter_config(C.CONFIGS[model](), in_channels)
    specs = {k[:-len(".weight")]: shape for k, shape, _ in T.t2i_adapter_param_specs(cfg) if k.endswith(".weight")}
    for h, w in P.T2I_ADAPTER_SIZES[model]:
        for B in P.T2I_ADAPTER_BATCHES:
            launches = TG.t2i_adapter_gemm_launches(cfg, 8 * h, 8 * w, B)
            names = [l["name"] for l in launches]
            assert sorted(names) == sorted(specs), f"{model} {h}x{w} B{B}: launches {names}, weights {sorted(specs)}"
            for l in launches:
                cout, cin, kh, kw = specs[l["name"]]
                if l["kind"] == "conv":
                    assert (kh, kw) == (3, 3) and (l["Cout"], 9 * l["Cin"], l["B"]) == (cout, 9 * cin, B), l["name"]
                else:
                    assert (kh, kw) == (1, 1) and (l["N"], l["K"]) == (cout, cin) and l["M"] % B == 0, l["name"]
                assert (l.get("addend") == "in_place") == l["name"].endswith(".block2"), l["name"]
            assert launches[0]["Cin"] == in_channels * cfg.downscale_factor ** 2
            assert launches[0]["H"] * cfg.downscale_factor == 8 * h


@pytest.mark.parametrize("model,E", sorted(REQUIRED_IP_PLUS))
def test_ip_plus_launches_match_resampler_shapes(model, E):
    """The Plus list's Resampler launches have the (N, K) of `resampler_shapes(plus_geometry(...), D)` for their weight
    keys (one layer stands for all, the layers' shapes are equal), over every weight matrix; to_kv_ip runs at
    M = NB·num_queries; there is no image_proj.proj."""
    from cfgpp_b200 import ip_adapter as IP
    cfg = C.CONFIGS[model]()
    g = IP.plus_geometry(cfg, E)
    shapes = IP.resampler_shapes(g, cfg.cross_attention_dim)
    mats = {k[:-len(".weight")] for k, s in shapes.items() if k.endswith(".weight") and len(s) == 2}
    T = IP.plus_encoder_config(cfg, E).num_positions
    for NB in P.IP_PLUS_NB:
        launches = [l for l in TG.ip_plus_launches(model, E) if l["name"].startswith(f"NB{NB} ")]
        names = {l["name"][len(f"NB{NB} "):]: l for l in launches}
        res = {n: l for n, l in names.items() if n.startswith("image_proj.")}
        assert set(res) == {m for m in mats if not m.startswith("image_proj.layers.") or ".layers.0." in m}
        for n, l in res.items():
            assert (l["N"], l["K"]) == shapes[n + ".weight"], n
            assert l["M"] == NB * (T + g["num_queries"] if n.endswith("to_kv") else
                                   T if n.endswith("proj_in") else g["num_queries"]), n
        kv = [l for n, l in names.items() if n.endswith(".attn2.to_kv_ip")]
        assert len(kv) == len(IP.processor_blocks(cfg))
        assert {l["M"] for l in kv} == {NB * g["num_queries"]}
    assert g["num_queries"] == 16 and T == 257


def test_adapter_lists_cover_their_edges():
    """The T2I lists hold an in-place residual, convolutions at the 96/48/24/12-wide levels (the im2col A tile) and
    both image batches; the Plus lists run to_kv_ip with 16 image tokens."""
    lists = TG.production_lists()
    t2i = [l for k, v in lists.items() if k[0] == "t2i_adapter" for _, l in v]
    assert any(l.get("addend") == "in_place" for l in t2i)
    convs = [l for l in t2i if l["kind"] == "conv"]
    assert {96, 48, 24, 12} <= {l["W"] for l in convs}
    assert {l["B"] for l in convs} == set(P.T2I_ADAPTER_BATCHES)
    plus = [l for k, v in lists.items() if k[0] == "ip_adapter_plus" for _, l in v]
    assert 4 * 16 in {l["M"] for l in plus if l["name"].endswith("to_kv_ip")}
