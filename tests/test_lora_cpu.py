"""LoRA on the host: the three file namings read back to the same adapter, literal known answers for the SGM block
numbering, every refusal, and the oracle's merge rule against the unmerged form. No GPU."""
import dataclasses
import math
import warnings

import pytest
import torch
from safetensors.torch import save_file

from cfgpp_b200 import config as C
from cfgpp_b200 import lora as L
from cfgpp_b200 import weights as Wt


def make_adapter(cfg, rank=2, seed=0, alpha=None, keys=None, dtype=torch.float16):
    """A random adapter on every weight of two or more dimensions (or on `keys`)."""
    g = torch.Generator().manual_seed(seed)
    targets = {}
    for key, shape, _ in Wt.unet_param_specs(cfg):
        if len(shape) < 2 or (keys is not None and key not in keys):
            continue
        N, K = shape[0], math.prod(shape[1:])
        down = (torch.randn(rank, K, generator=g) / math.sqrt(K)).to(dtype)
        up = (torch.randn(N, rank, generator=g) * 0.1).to(dtype)
        targets[key] = (down, up, float(rank if alpha is None else alpha))
    return targets


def to_file_dict(targets, cfg, naming, conv_4d=True):
    """The state dict a file of `naming` would hold."""
    shapes = {k: s for k, s, _ in Wt.unet_param_specs(cfg)}
    spell = L.module_spellings(cfg)
    out = {}
    for key, (down, up, alpha) in targets.items():
        stem = spell[key][naming]
        if conv_4d and len(shapes[key]) == 4:
            down = down.reshape(down.shape[0], *shapes[key][1:])
            up = up.reshape(*up.shape, 1, 1)
        if naming == "diffusers":
            out[f"unet.{stem}.lora_A.weight"], out[f"unet.{stem}.lora_B.weight"] = down, up
        else:
            out[f"{stem}.lora_down.weight"], out[f"{stem}.lora_up.weight"] = down, up
            out[f"{stem}.alpha"] = torch.tensor(alpha)
    return {k: v.contiguous() for k, v in out.items()}


@pytest.mark.parametrize("name", ["sd15", "sd2", "sdxl", "sdxl_refiner"])
@pytest.mark.parametrize("naming", L.NAMINGS)
def test_every_naming_round_trips_every_target(name, naming, tmp_path):
    cfg = C.CONFIGS[name]()
    targets = make_adapter(cfg, rank=1, alpha=1.0 if naming == "diffusers" else 0.5)
    path = tmp_path / "lora.safetensors"
    save_file(to_file_dict(targets, cfg, naming), str(path))
    back = L.read_lora(str(path), cfg)
    assert back.name == "lora" and not back.skipped_text_encoder
    assert set(back.targets) == set(targets) == {k for k, s, _ in Wt.unet_param_specs(cfg) if len(s) >= 2}
    for key, (down, up, alpha) in targets.items():
        d, u, a = back.targets[key]
        assert torch.equal(d, down) and torch.equal(u, up) and a == alpha, key


def test_spellings_are_unambiguous():
    for name in ("sd15", "sdxl", "sdxl_refiner", "tiny_sdxl", "tiny_sd15"):
        cfg = C.CONFIGS[name]()
        spell = L.module_spellings(cfg)
        for naming in L.NAMINGS:
            stems = [s[naming] for s in spell.values()]
            assert len(set(stems)) == len(stems), (name, naming)


SDXL_SGM = {
    "input_blocks_0_0": "conv_in.weight",
    "input_blocks_4_1_transformer_blocks_0_attn1_to_q": "down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q.weight",
    "input_blocks_3_0_op": "down_blocks.0.downsamplers.0.conv.weight",
    "input_blocks_1_0_in_layers_2": "down_blocks.0.resnets.0.conv1.weight",
    "input_blocks_8_1_transformer_blocks_9_ff_net_0_proj": "down_blocks.2.attentions.1.transformer_blocks.9.ff.net.0.proj.weight",
    "middle_block_1_proj_in": "mid_block.attentions.0.proj_in.weight",
    "middle_block_2_emb_layers_1": "mid_block.resnets.1.time_emb_proj.weight",
    "output_blocks_2_2_conv": "up_blocks.0.upsamplers.0.conv.weight",
    "output_blocks_0_0_skip_connection": "up_blocks.0.resnets.0.conv_shortcut.weight",
    "output_blocks_5_1_transformer_blocks_1_attn2_to_out_0": "up_blocks.1.attentions.2.transformer_blocks.1.attn2.to_out.0.weight",
    "output_blocks_8_0_out_layers_3": "up_blocks.2.resnets.2.conv2.weight",
    "time_embed_0": "time_embedding.linear_1.weight",
    "label_emb_0_2": "add_embedding.linear_2.weight",
    "out_2": "conv_out.weight",
}


@pytest.mark.parametrize("stem,key", sorted(SDXL_SGM.items()))
def test_sgm_numbering_known_answers_sdxl(stem, key):
    cfg = C.CONFIGS["sdxl"]()
    shape = {k: s for k, s, _ in Wt.unet_param_specs(cfg)}[key]
    sd = {f"lora_unet_{stem}.lora_down.weight": torch.zeros(4, math.prod(shape[1:])),
          f"lora_unet_{stem}.lora_up.weight": torch.zeros(shape[0], 4), f"lora_unet_{stem}.alpha": torch.tensor(2.0)}
    ad = L.read_lora(sd, cfg)
    assert list(ad.targets) == [key] and ad.targets[key][2] == 2.0 and ad.targets[key][0].dtype == torch.float16


def test_sgm_numbering_known_answers_sd15():
    cfg = C.CONFIGS["sd15"]()
    spell = L.module_spellings(cfg)
    assert spell["up_blocks.0.upsamplers.0.conv.weight"]["kohya_sgm"] == "lora_unet_output_blocks_2_1_conv"
    assert spell["up_blocks.1.upsamplers.0.conv.weight"]["kohya_sgm"] == "lora_unet_output_blocks_5_2_conv"
    assert spell["down_blocks.3.resnets.1.conv1.weight"]["kohya_sgm"] == "lora_unet_input_blocks_11_0_in_layers_2"
    assert spell["down_blocks.2.downsamplers.0.conv.weight"]["kohya_sgm"] == "lora_unet_input_blocks_9_0_op"
    assert (spell["down_blocks.0.attentions.1.proj_out.weight"]["kohya_sgm"] == "lora_unet_input_blocks_2_1_proj_out")


def test_older_diffusers_spellings_and_alpha_default():
    cfg = C.tiny_sdxl_config()
    key = next(k for k, _, _ in Wt.unet_param_specs(cfg) if k.endswith("attn1.to_q.weight"))
    out_key = key.replace("to_q", "to_out.0")
    c = {k: s for k, s, _ in Wt.unet_param_specs(cfg)}[key][0]
    mod, block = key[:-len(".weight")], key[:-len(".to_q.weight")]
    d, u = torch.randn(3, c), torch.randn(c, 3)
    for sd in ({f"{mod}.lora.down.weight": d, f"{mod}.lora.up.weight": u},
               {f"unet.{block}.processor.to_q_lora.down.weight": d, f"unet.{block}.processor.to_q_lora.up.weight": u}):
        ad = L.read_lora(sd, cfg)
        assert list(ad.targets) == [key] and ad.targets[key][2] == 3.0  # alpha absent: alpha = rank
        assert torch.equal(ad.targets[key][0], d.half()) and torch.equal(ad.targets[key][1], u.half())
    ad = L.read_lora({f"{block}.processor.to_out_lora.down.weight": d, f"{block}.processor.to_out_lora.up.weight": u},
                     cfg, alpha=6.0)
    assert list(ad.targets) == [out_key] and ad.targets[out_key][2] == 6.0


def _one(cfg, suffix="attn2.to_k.weight"):
    key = next(k for k, _, _ in Wt.unet_param_specs(cfg) if k.endswith(suffix))
    shape = {k: s for k, s, _ in Wt.unet_param_specs(cfg)}[key]
    return key, shape, L.module_spellings(cfg)[key]["kohya"]


def test_refusals_name_the_key():
    cfg = C.tiny_sdxl_config()
    key, shape, stem = _one(cfg)
    N, K = shape[0], math.prod(shape[1:])
    good = {f"{stem}.lora_down.weight": torch.zeros(4, K), f"{stem}.lora_up.weight": torch.zeros(N, 4)}
    L.read_lora(good, cfg)
    for extra in ("dora_scale", "hada_w1_a", "lokr_w1", "lora_mid.weight"):
        with pytest.raises(ValueError, match=f"{stem}.{extra}"):
            L.read_lora({**good, f"{stem}.{extra}": torch.zeros(1)}, cfg)
    with pytest.raises(ValueError, match="rank 129"):
        L.read_lora({f"{stem}.lora_down.weight": torch.zeros(129, K), f"{stem}.lora_up.weight": torch.zeros(N, 129)}, cfg)
    with pytest.raises(ValueError, match=f"{stem}.*do not fit.*{key}"):
        L.read_lora({f"{stem}.lora_down.weight": torch.zeros(4, K + 1), f"{stem}.lora_up.weight": torch.zeros(N, 4)}, cfg)
    with pytest.raises(ValueError, match=f"{stem}.*do not fit"):
        L.read_lora({f"{stem}.lora_down.weight": torch.zeros(4, K), f"{stem}.lora_up.weight": torch.zeros(N, 5)}, cfg)
    with pytest.raises(ValueError, match="lora_unet_no_such_module.*maps to no weight"):
        L.read_lora({"lora_unet_no_such_module.lora_down.weight": torch.zeros(4, 4)}, cfg)
    with pytest.raises(ValueError, match="lacks its up factor"):
        L.read_lora({f"{stem}.lora_down.weight": torch.zeros(4, K)}, cfg)
    ckey, cshape, cstem = _one(cfg, "resnets.0.conv1.weight")
    with pytest.raises(ValueError, match=f"{cstem}.lora_up.weight.*3x3 kernel"):
        L.read_lora({f"{cstem}.lora_down.weight": torch.zeros(4, cshape[1], 1, 1),
                     f"{cstem}.lora_up.weight": torch.zeros(cshape[0], 4, 3, 3)}, cfg)
    with pytest.raises(ValueError, match="norm1"):  # a 1-D parameter is no target
        L.read_lora({"lora_unet_mid_block_resnets_0_norm1.lora_down.weight": torch.zeros(4, 4)}, cfg)


def test_text_encoder_entries_warn_once_and_are_kept_aside():
    cfg = C.tiny_sdxl_config()
    key, shape, stem = _one(cfg)
    sd = {f"{stem}.lora_down.weight": torch.zeros(4, shape[1]), f"{stem}.lora_up.weight": torch.zeros(shape[0], 4),
          "lora_te1_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": torch.zeros(4, 8),
          "lora_te1_text_model_encoder_layers_0_mlp_fc1.lora_up.weight": torch.zeros(8, 4),
          "text_encoder.text_model.encoder.layers.0.self_attn.q_proj.lora_A.weight": torch.zeros(4, 8)}
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        ad = L.read_lora(sd, cfg)
    assert len(w) == 1 and "text-encoder" in str(w[0].message)
    assert list(ad.targets) == [key] and len(ad.skipped_text_encoder) == 3
    assert L.is_lora_keys(sd) and not L.is_lora_keys(k for k, _, _ in Wt.unet_param_specs(cfg))


def test_fp32_and_bf16_factors_round_once_to_fp16():
    cfg = C.tiny_sd15_config()
    key, shape, stem = _one(cfg)
    d = torch.randn(2, shape[1])
    for dt in (torch.float32, torch.bfloat16):
        ad = L.read_lora({f"{stem}.lora_down.weight": d.to(dt), f"{stem}.lora_up.weight": torch.ones(shape[0], 2, dtype=dt)}, cfg)
        assert torch.equal(ad.targets[key][0], d.to(dt).to(torch.float16))


# ---- oracle -----------------------------------------------------------------------------------------------------
def _oracle_pair(name, seed=5):
    from oracle import unet as O
    cfg = C.CONFIGS[name]()
    sd = Wt.synthetic_state_dict(cfg, seed=seed, device="cpu")
    ocfg = O.UNetConfig(**{f.name: getattr(cfg, f.name) for f in dataclasses.fields(O.UNetConfig)})
    return cfg, sd, ocfg, O


def _forward(m, cfg, seed=3):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(2, 4, 16, 16, generator=g, dtype=torch.float64)
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=g, dtype=torch.float64)
    add = None
    if cfg.addition_embed_type == "text_time":
        add = {"text_embeds": torch.randn(2, cfg.pooled_dim, generator=g, dtype=torch.float64),
               "time_ids": torch.tensor([[128., 128, 0, 0, 128, 128]] * 2, dtype=torch.float64)}
    with torch.no_grad():
        return m(z, torch.tensor(500), ctx, add)["sample"]


@pytest.mark.parametrize("name", ["tiny_sdxl", "tiny_sd15"])
def test_oracle_merged_equals_unmerged(name):
    """The merge rule is the formula a LoRA trainer optimises: base(x) + c up(down(x)) on every Linear and Conv2d."""
    from oracle import lora as OL
    cfg, sd, ocfg, O = _oracle_pair(name)
    a1, a2 = make_adapter(cfg, rank=3, seed=1, alpha=1.5), make_adapter(cfg, rank=2, seed=2)
    scales = [0.8, -0.5]
    merged = OL.merge_state_dict({k: v.double() for k, v in sd.items()}, [a1, a2], scales, dtype=torch.float64)
    y_m = _forward(O.build_unet(ocfg, merged, dtype=torch.float64), cfg)
    y_u = _forward(OL.attach(O.build_unet(ocfg, sd, dtype=torch.float64), [a1, a2], scales), cfg)
    y_0 = _forward(O.build_unet(ocfg, sd, dtype=torch.float64), cfg)
    err = ((y_m - y_u).norm() / y_u.norm()).item()
    moved = ((y_0 - y_u).norm() / y_u.norm()).item()
    print(f"{name}: merged vs unmerged rel-L2 {err:.2e}; adapter moved the output by {moved:.2e}")
    assert err <= 1e-5 and moved > 1e-2


def test_oracle_merge_rule():
    from oracle import lora as OL
    cfg = C.tiny_sdxl_config()
    sd = Wt.synthetic_state_dict(cfg, seed=5, device="cpu")
    a1, a2 = make_adapter(cfg, rank=4, seed=1, alpha=2.0), make_adapter(cfg, rank=4, seed=2)
    zero = OL.merge_state_dict(sd, [a1, a2], [0.0, 0.0])
    assert all(torch.equal(zero[k], sd[k]) for k in sd)  # scale 0: the input bit for bit
    key = "mid_block.attentions.0.transformer_blocks.0.attn1.to_v.weight"
    both = OL.merge_state_dict(sd, [a1, a2], [1.0, 0.25])[key]
    d1, u1, _ = a1[key]
    d2, u2, _ = a2[key]
    want = (sd[key].double() + 0.5 * (u1.double() @ d1.double()) + 0.25 * (u2.double() @ d2.double())).half()
    assert torch.equal(both, want)  # alpha / r = 2 / 4; alpha default = r; two adapters add
    assert both.dtype == torch.float16 and not torch.equal(both, sd[key])
    untouched = OL.merge_state_dict(sd, [{key: a1[key]}], [1.0])
    assert all(torch.equal(untouched[k], sd[k]) for k in sd if k != key)
