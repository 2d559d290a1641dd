"""LoRA on the device: the merge kernel per element against fp64, the refresh of every packed layout bit for bit, no
drift over scale switches, the plan and graph surviving a switch, and the solver surface.

The merge rule: out = fp16( fp32(base) + sum_a c_a * acc_a ), acc_a the fp32 tensor-core sum of exact fp16 x fp16
products over rank r_a. Against the exact value ref (fp64) the error of one element is bounded by

    E = 1/2 ulp_fp16(|ref| + e32) + e32
    e32 = sum_a |c_a| (r_a + 2) 2^-22 A_a  +  (n_adapters + 1) 2^-23 (|base| + sum_a |c_a| A_a),   A_a = sum_r |up||down|

the first term of e32 covering the fp32 accumulation of r_a products on the tensor cores (which may truncate rather
than round: 2^-22 per add instead of 2^-24) and the multiplication by c_a, the second the fp32 adds that combine the
adapters with the base; the half ulp is the single rounding to fp16. The largest |err| / E is printed.
"""
import math
from types import SimpleNamespace

import pytest
import torch
from safetensors.torch import save_file

from cfgpp_b200 import _native as nv
from cfgpp_b200 import config as C
from cfgpp_b200 import lora as L
from cfgpp_b200 import weights as Wt
from cfgpp_b200.engine import NativeUNet
from helpers import OracleCudaUNet, make_inputs, oracle_cfg, rel_l2
from oracle import lora as OL

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
MSG = "call cfgpp_set_prompt again"


# ---- helpers ------------------------------------------------------------------------------------------------------
def ulp16(x):
    x = x.abs().clamp(min=2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(x)) - 10)


def merge_bound(base, downs, ups, coefs):
    ref = base.double()
    mag = base.double().abs()
    e32 = torch.zeros_like(ref)
    for d, u, c in zip(downs, ups, coefs):
        ref = ref + c * (u.double() @ d.double())
        A = abs(c) * (u.double().abs() @ d.double().abs())
        e32 += (d.shape[0] + 2) * 2.0 ** -22 * A
        mag = mag + A
    e32 += (len(downs) + 1) * 2.0 ** -23 * mag
    return ref, 0.5 * ulp16(ref.abs() + e32) + e32


def check_merge(base, downs, ups, coefs, label):
    out = nv.op_lora_merge(base, downs, ups, coefs)
    ref, E = merge_bound(base, downs, ups, coefs)
    over = ref.abs() + E >= 65520.0  # rounds to +-inf: checked by sign below
    o = out.double()
    assert torch.isfinite(o[~over]).all(), label
    worst = ((o - ref).abs() / E)[~over].max().item() if (~over).any() else 0.0
    print(f"lora merge {label}: N={base.shape[0]} K={base.shape[1]} ranks={[d.shape[0] for d in downs]} "
          f"max |err|/E = {worst:.3f}")
    assert worst <= 1.0, label
    sure = ref.abs() - E >= 65520.0
    assert torch.equal(torch.isinf(out[sure]), torch.ones_like(out[sure], dtype=torch.bool)), label
    assert torch.equal(torch.sign(out[sure].float()), torch.sign(ref[sure]).float()), label
    return out


def rand_factors(N, K, ranks, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    downs = [(torch.randn(r, K, generator=g) * scale).half().to(dev) for r in ranks]
    ups = [torch.randn(N, r, generator=g).half().to(dev) for r in ranks]
    return downs, ups


def exact_adapter(cfg, seed, keys=None):
    """One non-zero power of two per row of `up`, down in {-2..2} * 2^-9, alpha / r = 1 / 2: every product, the scaled sum and
    fp32(W) + delta are exact, so the device merge and the fp64 rule round the same number once."""
    g = torch.Generator().manual_seed(seed)
    targets = {}
    for key, shape, _ in Wt.unet_param_specs(cfg):
        if len(shape) < 2 or (keys is not None and not keys(key)):
            continue
        N, K, r = shape[0], math.prod(shape[1:]), 4
        down = torch.randint(-2, 3, (r, K), generator=g).float() * 2.0 ** -9
        up = torch.zeros(N, r)
        up[torch.arange(N), torch.randint(0, r, (N,), generator=g)] = \
            torch.exp2(-torch.randint(1, 4, (N,), generator=g).float()) * (torch.randint(0, 2, (N,), generator=g) * 2 - 1)
        targets[key] = (down.half(), up.half(), 2.0)  # alpha / r = 1 / 2
    return L.LoraAdapter(targets)


def random_adapter(cfg, rank, seed, keys=None, gain=0.3):
    g = torch.Generator().manual_seed(seed)
    targets = {}
    for key, shape, _ in Wt.unet_param_specs(cfg):
        if len(shape) < 2 or (keys is not None and not keys(key)):
            continue
        N, K = shape[0], math.prod(shape[1:])
        down = torch.randn(rank, K, generator=g) / math.sqrt(K)
        up = torch.randn(N, rank, generator=g) * (gain / math.sqrt(rank))
        targets[key] = (down.half(), up.half(), float(rank))
    return L.LoraAdapter(targets)


def build(name, seed=1234, sd=None):
    cfg = C.CONFIGS[name]()
    sd = sd if sd is not None else Wt.synthetic_state_dict(cfg, seed=seed, device=dev)
    return cfg, sd, NativeUNet(cfg, sd, dev)


def forward(net, cfg, B=1, hw=32, t=500.0, seed=7):
    z, uc, c, add = make_inputs(cfg, B, hw, dev, seed=seed)
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"] if add else None, add["time_ids"].float() if add else None)
    return torch.cat(net.predict_noise(z, t))


# ---- 1 / 2: the merge kernel --------------------------------------------------------------------------------------
@pytest.mark.parametrize("rank", [1, 3, 4, 8, 16, 17, 64, 128])
def test_merge_kernel_ranks(rank):
    g = torch.Generator().manual_seed(rank)
    for N, K in ((320, 320), (100, 136), (77, 45)):
        base = torch.randn(N, K, generator=g).half().to(dev)
        downs, ups = rand_factors(N, K, [rank], rank)
        check_merge(base, downs, ups, [0.7], f"rank {rank}")


@pytest.mark.parametrize("N,K", [(4, 2880), (320, 36), (4, 36), (64, 2560 * 9), (1, 1), (65, 63), (129, 8)])
def test_merge_kernel_ragged_shapes(N, K):
    g = torch.Generator().manual_seed(N * 7 + K)
    base = torch.randn(N, K, generator=g).half().to(dev)
    downs, ups = rand_factors(N, K, [5, 16], N + K, scale=0.1)
    check_merge(base, downs, ups, [1.0, -0.25], "ragged")


@pytest.mark.parametrize("n_adapters", [0, 1, 2, 3, 4])
def test_merge_kernel_adapter_counts_and_signs(n_adapters):
    g = torch.Generator().manual_seed(n_adapters)
    base = torch.randn(200, 264, generator=g).half().to(dev)
    ranks = [8, 3, 64, 17][:n_adapters]
    coefs = [0.8, -1.5, 0.0, 0.125][:n_adapters]
    downs, ups = rand_factors(200, 264, ranks, 11, scale=0.2)
    out = check_merge(base, downs, ups, coefs, f"{n_adapters} adapters")
    if n_adapters == 0:
        assert torch.equal(out, base)
    zero = nv.op_lora_merge(base, downs, ups, [0.0] * n_adapters)
    assert torch.equal(zero, base)  # all scales zero: the base bits
    d5, u5 = rand_factors(200, 264, [1] * 5, 12)
    with pytest.raises(nv.NativeError, match="at most 4"):
        nv.op_lora_merge(base, d5, u5, [1.0] * 5)


def test_merge_kernel_extreme_bases_and_overflow():
    g = torch.Generator().manual_seed(5)
    N, K = 96, 128
    downs, ups = rand_factors(N, K, [16], 3)
    big = (torch.rand(N, K, generator=g) * 5000 + 60000).half() * (torch.randint(0, 2, (N, K), generator=g) * 2 - 1).half()
    check_merge(big.to(dev), downs, ups, [1.0], "base near fp16 max")
    sub = (torch.randint(-1023, 1024, (N, K), generator=g).float() * 2.0 ** -24).half().to(dev)
    tiny_d = [(d.float() * 2.0 ** -12).half() for d in downs]
    check_merge(sub, tiny_d, ups, [2.0 ** -6], "subnormal base and result")
    # far past the largest finite fp16: +-inf with the sign of the exact value
    d1 = [torch.full((1, K), 100.0).half().to(dev)]
    u1 = [(torch.arange(N).float() - N / 2 + 0.5).sign().mul(200.0).half().reshape(N, 1).to(dev)]
    out = check_merge(big.to(dev) * 0 + 60000 * u1[0].sign(), d1, u1, [1.0], "overflow")
    assert torch.isinf(out).all()


def test_merge_kernel_integer_known_answers():
    g = torch.Generator().manual_seed(9)
    for N, K, ranks, coefs in ((64, 64, [16], [0.5]), (130, 200, [3, 128], [2.0, -0.25]), (4, 36, [1, 4, 8, 17], [1.0, 0.5, -1.0, 4.0])):
        base = torch.randint(-64, 65, (N, K), generator=g).half().to(dev)
        downs = [torch.randint(-2, 3, (r, K), generator=g).half().to(dev) for r in ranks]
        ups = [torch.randint(-2, 3, (N, r), generator=g).half().to(dev) for r in ranks]
        want = base.double()
        for d, u, c in zip(downs, ups, coefs):
            want = want + c * (u.double() @ d.double())
        assert want.abs().max() < 2048
        got = nv.op_lora_merge(base, downs, ups, coefs)
        assert torch.equal(got.double(), want)


# ---- 3: every packed layout is refreshed, bit for bit ---------------------------------------------------------------
GROUPS = {
    "conv3x3": lambda k: ".resnets." in k and (k.endswith("conv1.weight") or k.endswith("conv2.weight")),
    "resampler conv": lambda k: "samplers" in k,
    "1x1 shortcut": lambda k: "conv_shortcut" in k,
    "proj_in": lambda k: k.endswith("proj_in.weight"),
    "proj_out": lambda k: k.endswith("proj_out.weight"),
    "self q|k|v": lambda k: ".attn1.to_" in k and "to_out" not in k,
    "self v only": lambda k: k.endswith("attn1.to_v.weight"),
    "cross to_q": lambda k: k.endswith("attn2.to_q.weight"),
    "cross k|v": lambda k: k.endswith("attn2.to_k.weight") or k.endswith("attn2.to_v.weight"),
    "cross v only": lambda k: k.endswith("attn2.to_v.weight"),
    "to_out": lambda k: "to_out.0.weight" in k,
    "geglu": lambda k: k.endswith("ff.net.0.proj.weight"),
    "ff.net.2": lambda k: k.endswith("ff.net.2.weight"),
    "time_emb_proj": lambda k: "time_emb_proj" in k,
    "time_embedding": lambda k: k.startswith("time_embedding"),
    "add_embedding": lambda k: k.startswith("add_embedding"),
    "conv_in": lambda k: k == "conv_in.weight",
    "conv_out": lambda k: k == "conv_out.weight",
    "every weight": lambda k: True,
}


@pytest.mark.parametrize("name", ["tiny_sdxl", "tiny_sd15"])
def test_adapter_reaches_every_packed_layout(name):
    cfg, sd, a = build(name)
    base_out = forward(a, cfg)
    all_keys = [k for k, s, _ in Wt.unet_param_specs(cfg) if len(s) >= 2]
    seen = set()
    for i, (group, pick) in enumerate(GROUPS.items()):
        if not any(pick(k) for k in all_keys):
            assert group in ("add_embedding", "1x1 shortcut"), group  # not in this architecture
            continue
        ad = exact_adapter(cfg, seed=100 + i, keys=pick)
        seen |= set(ad.targets)
        a.clear_lora()
        a.add_lora(ad, 0.5)
        got = forward(a, cfg)
        merged = OL.merge_state_dict(sd, [ad.targets], [0.5])
        assert any(not torch.equal(merged[k], sd[k]) for k in ad.targets)
        _, _, b = build(name, sd=merged)
        want = forward(b, cfg)
        b.close()
        assert torch.equal(got, want), f"{name}: adapter on {group} differs from the host-merged weights"
        assert not torch.equal(got, base_out), f"{name}: adapter on {group} did not change the output"
        stats = a.lora_stats
        assert stats["targets"] == len(ad.targets) and stats["adapters"] == 1
        assert stats["backup_bytes"] == sum(2 * sd[k].numel() for k in ad.targets)
        assert stats["bytes_moved"] >= 2 * stats["backup_bytes"]
    assert seen == set(all_keys)
    a.clear_lora()
    assert torch.equal(forward(a, cfg), base_out) and a.lora_stats["backup_bytes"] == 0
    a.close()


def test_second_size_prepared_with_adapter_on():
    """A plan built after the merge packs the merged weights: raw storage holds W_eff."""
    cfg, sd, a = build("tiny_sd15")
    ad = exact_adapter(cfg, seed=3)
    a.add_lora(ad, 1.0)
    got32, got16 = forward(a, cfg, hw=32), forward(a, cfg, B=2, hw=16)
    _, _, b = build("tiny_sd15", sd=OL.merge_state_dict(sd, [ad.targets], [1.0]))
    assert torch.equal(got32, forward(b, cfg, hw=32)) and torch.equal(got16, forward(b, cfg, B=2, hw=16))
    a.close(), b.close()


def test_native_refusals_name_the_key():
    cfg, sd, a = build("tiny_sdxl")
    key = "mid_block.attentions.0.proj_in.weight"
    ads = [exact_adapter(cfg, seed=s, keys=lambda k: k == key) for s in range(5)]
    for ad in ads[:4]:
        a.add_lora(ad, 1.0)
    with pytest.raises(ValueError, match=key):
        a.add_lora(ads[4], 1.0)
    assert a.lora_stats["adapters"] == 4 and list(a.loras) == ["lora0", "lora1", "lora2", "lora3"]
    d, u, _ = ads[0].targets[key]
    st = nv.stream_ptr()
    from ctypes import c_float, c_int
    for bad_key, rank, msg in (("no.such.weight", 4, "no.such.weight"), ("conv_in.bias", 4, "conv_in.bias"), (key, 129, key)):
        rc = a.lib.cfgpp_lora_add(a._h, c_int(4), bad_key.encode(), nv.ptr(d.to(dev)), nv.ptr(u.to(dev)), c_int(rank),
                                  c_float(1.0), c_int(0), st)
        assert rc != 0 and msg in a.lib.cfgpp_last_error().decode()
    with pytest.raises(KeyError):
        a.set_lora_scales({"nope": 1.0})
    a.close()


# ---- 4: random adapters at full size ------------------------------------------------------------------------------
@pytest.mark.parametrize("name,rank,keys,hw,t", [("sdxl", 16, lambda k: ".attn" in k, 128, 501), ("sd15", 8, None, 64, 401)])
def test_random_adapter_full_size_against_unmerged_oracle(name, rank, keys, hw, t):
    from oracle import unet as O
    cfg, sd, net = build(name)
    ad = random_adapter(cfg, rank, seed=21, keys=keys)
    z, uc, c, add = make_inputs(cfg, 1, hw, dev)
    net.prepare(1, hw, hw)
    set_prompt = lambda: net.set_prompt(torch.cat([uc, c]), add["text_embeds"] if add else None,  # noqa: E731
                                        add["time_ids"].float() if add else None)
    set_prompt()
    base = torch.cat(net.predict_noise(z, float(t))).float()
    net.add_lora(ad, 0.9)
    set_prompt()
    got = torch.cat(net.predict_noise(z, float(t))).float()
    net.close()
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
    ref16 = OracleCudaUNet(cfg, sd, dev)
    OL.attach(ref16.m, [ad.targets], [0.9])
    r16 = ref16(z_in, t_in, ctx, add)["sample"].float()
    del ref16
    m32 = OL.attach(O.build_unet(oracle_cfg(cfg), sd, dtype=torch.float32, device=dev), [ad.targets], [0.9])
    with torch.no_grad():
        r32 = m32(z_in, t_in, ctx.float(), {k: v.float() for k, v in add.items()} if add else None)["sample"]
    del m32
    e16, e32, o32 = rel_l2(got, r16), rel_l2(got, r32), rel_l2(r16, r32)
    print(f"{name} rank {rank}: rel-L2 vs fp16 unmerged oracle {e16:.3e}, vs fp32 {e32:.3e} (fp16 oracle's own {o32:.3e}); "
          f"adapter moved the output by {rel_l2(got, base):.3e}")
    assert rel_l2(got, base) > 1e-2
    assert e16 <= 5e-3 and e32 <= 1.5 * o32 + 1e-4


# ---- 5: no drift ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny_sdxl", "tiny_sd15"])
def test_scale_switches_do_not_drift(name):
    cfg, sd, a = build(name)
    untouched = forward(a, cfg)
    ad1, ad2 = random_adapter(cfg, 8, seed=1), random_adapter(cfg, 5, seed=2, keys=lambda k: ".attn" in k)
    n1, n2 = a.add_lora(ad1, 0.8), a.add_lora(ad2, 0.4)
    first = forward(a, cfg)
    for s in (0.3, 1.7, -0.6):
        a.set_lora_scales({n1: s})
    a.set_lora_scales({n1: 0.8})
    again = forward(a, cfg)
    _, _, fresh = build(name)
    fresh.add_lora(ad1, 0.8), fresh.add_lora(ad2, 0.4)
    want = forward(fresh, cfg)
    fresh.close()
    assert torch.equal(first, want) and torch.equal(again, want) and not torch.equal(want, untouched)
    a.set_lora_scales({n1: 0.0, n2: 0.0})
    assert torch.equal(forward(a, cfg), untouched) and a.lora_stats["backup_bytes"] > 0
    a.set_lora_scales({n1: 0.8, n2: 0.4})
    a.clear_lora()
    assert torch.equal(forward(a, cfg), untouched)
    assert a.lora_stats == {"adapters": 0, "targets": 0, "backup_bytes": 0, "bytes_moved": a.lora_stats["bytes_moved"]}
    assert a.loras == {}
    a.close()


# ---- 6: the plan and the graph survive ----------------------------------------------------------------------------------
def test_plan_and_graph_survive_a_switch():
    from cfgpp_b200 import schedule as S
    cfg, sd, a = build("tiny_sdxl")
    z, uc, c, add = make_inputs(cfg, 1, 32, dev)
    steps = S.ddim_cfgpp_steps(S.Schedule.make(6), 0.6, True)

    def trajectory(net, rebind=True):
        if rebind:
            net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
        net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
        net.set_state(z)
        net.run_steps()
        return net.get_state(0)

    a.prepare(1, 32, 32)
    before = (a.launches_per_step, a.plan_stats, a.workspace_bytes)
    z_base = trajectory(a)
    ad = random_adapter(cfg, 8, seed=4)
    name = a.add_lora(ad, 0.8)
    assert (a.launches_per_step, a.plan_stats, a.workspace_bytes) == before
    with pytest.raises(nv.NativeError, match=MSG):
        trajectory(a, rebind=False)
    with pytest.raises(nv.NativeError, match=MSG):
        a.predict_noise(z, 500.0)
    z_08 = trajectory(a)
    a.set_lora_scales({name: 0.3})
    with pytest.raises(nv.NativeError, match=MSG):
        a.run_steps()
    z_03 = trajectory(a)
    _, _, f = build("tiny_sdxl")
    f.add_lora(ad, 0.3)
    f.prepare(1, 32, 32)
    assert torch.equal(z_03, trajectory(f))
    f.set_lora_scales({"lora0": 0.8})
    assert torch.equal(z_08, trajectory(f)) and not torch.equal(z_08, z_base) and not torch.equal(z_08, z_03)
    a.clear_lora()
    with pytest.raises(nv.NativeError, match=MSG):
        a.run_steps()
    assert torch.equal(trajectory(a), z_base)
    a.close(), f.close()


# ---- 7: solvers ------------------------------------------------------------------------------------------------------------
def _sample(solver, family, **kw):
    from cfgpp_b200.utils.log_util import set_seed
    set_seed(42)
    if family == "sdxl":
        return solver.sample(prompt1=["", "a cat"], prompt2=["", "a cat"], target_size=(256, 256), **kw)
    return solver.sample(prompt=["", "a cat"], **kw)


@pytest.mark.parametrize("family,method,cfg_name,lam", [("sdxl", "ddim_cfg++", "tiny_sdxl", 0.6),
                                                       ("sd", "dpm++_2m_cfg++", "tiny_sd15", 0.6),
                                                       ("sd", "ddim", "tiny_sd2", 5.0)])
def test_solver_load_lora(family, method, cfg_name, lam, tmp_path):
    from cfgpp_b200 import latent_diffusion as LD, latent_sdxl as LX
    cfg = getattr(C, cfg_name + "_config")()
    reg = LX if family == "sdxl" else LD
    kw = dict(solver_config=SimpleNamespace(num_sampling=5), device="cuda:0", unet_config=cfg,
              model_key=f"synthetic:73{len(method)}")
    s, twin = reg.get_solver(method, **kw), reg.get_solver(method, **kw)
    base = _sample(s, family, cfg_guidance=lam)
    ad = random_adapter(cfg, 4, seed=8)
    path = tmp_path / "style.safetensors"
    spell = L.module_spellings(cfg)
    save_file({f"{spell[k]['kohya_sgm']}.{part}": v.contiguous() for k, (d, u, al) in ad.targets.items()
               for part, v in (("lora_down.weight", d), ("lora_up.weight", u), ("alpha", torch.tensor(al)))}, str(path))
    name = s.load_lora(str(path), scale=0.7)
    assert name == "style" and dict(s.loras) == {"style": 0.7} == dict(twin.loras) and twin.unet is s.unet
    with pytest.raises(TypeError):
        s.loras["style"] = 1.0
    fused = _sample(s, family, cfg_guidance=lam)
    seen = []
    cb = _sample(s, family, cfg_guidance=lam, callback_fn=lambda i, t, kw: (seen.append(i), kw)[1])
    assert seen and torch.equal(fused, cb) and not torch.equal(fused, base) and torch.isfinite(fused).all()
    s.set_lora_scale("style", 0.2)
    assert dict(twin.loras) == {"style": 0.2} and not torch.equal(_sample(twin, family, cfg_guidance=lam), fused)
    s.set_lora_scale("style", 0.7)
    assert torch.equal(_sample(twin, family, cfg_guidance=lam), fused)
    s.unload_lora()
    assert dict(twin.loras) == {} and torch.equal(_sample(s, family, cfg_guidance=lam), base)


def test_lightning_from_a_lora_file_equals_the_merged_unet(tmp_path):
    from cfgpp_b200 import latent_sdxl as LX
    cfg = C.tiny_sdxl_config()
    ad = exact_adapter(cfg, seed=12)
    spell = L.module_spellings(cfg)
    lora_path, full_path = tmp_path / "lightning_lora.safetensors", tmp_path / "lightning_unet.safetensors"
    save_file({f"unet.{spell[k]['diffusers']}.{part}": v.contiguous() for k, (d, u, _) in ad.targets.items()
               for part, v in (("lora_A.weight", d), ("lora_B.weight", u))}, str(lora_path))
    sd = Wt.synthetic_state_dict(cfg, seed=7412, device=dev)  # what model_key "synthetic:7412" resolves to
    as_read = {k: (d, u, float(d.shape[0])) for k, (d, u, _) in ad.targets.items()}  # the file carries no alpha: alpha = r
    save_file({k: v.cpu().contiguous() for k, v in OL.merge_state_dict(sd, [as_read], [1.0]).items()}, str(full_path))
    kw = dict(solver_config=SimpleNamespace(num_sampling=4), device="cuda:0", unet_config=cfg)
    a = LX.get_solver("ddim_cfg++_lightning", base_model_key="synthetic:7412", light_model_ckpt=str(lora_path), **kw)
    b = LX.get_solver("ddim_cfg++_lightning", light_model_ckpt=str(full_path), **kw)
    plain = LX.get_solver("ddim_cfg++", model_key="synthetic:7412", **kw)
    assert list(a.loras.values()) == [1.0] and dict(b.loras) == {} and dict(plain.loras) == {}  # its own engine
    assert a.unet is not plain.unet
    ia, ib = _sample(a, "sdxl", cfg_guidance=1.0), _sample(b, "sdxl", cfg_guidance=1.0)
    assert torch.equal(ia, ib) and not torch.equal(ia, _sample(plain, "sdxl", cfg_guidance=1.0))
