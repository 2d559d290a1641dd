"""The SDXL refiner on the GPU: the native add-embedding with a derived time-id count (a geometry that does not divide is
refused; 5 ids against the oracle), the refiner UNet at its real widths against the oracle, split base -> refiner
trajectories against the oracle's stated split rule, the same-weights identity (a "refiner" that is the base gives the
unsplit trajectory bit for bit), fused == callback across the hand-off, batched `sample()` with a refiner, and
`examples.text_to_img --model sdxl --denoising_end 0.8`. Every test prints what it measured (`pytest -s`).

Stated tolerances: UNet rel-L2 <= 5e-3 against the fp16-autocast oracle and an fp32 error <= 1.5x the fp16 oracle's
own (DESIGN section 3); teacher-forced step <= 5e-3, free-running final latent <= 3e-2; batch vs serial <= 3e-2."""
import dataclasses
import gc
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from helpers import OracleCudaUNet, oracle_cfg, rel_l2

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
ROOT = Path(__file__).resolve().parent.parent


class LatentVAE:
    """Stand-in VAE that keeps the latent it is asked to decode (the tests compare final latents)."""
    def __init__(self):
        self.latents = []

    def decode(self, z):
        self.latents.append(z.detach().clone())
        return torch.zeros(z.shape[0], 3, 8 * z.shape[2], 8 * z.shape[3], device=z.device)

    def encode(self, x, dtype=torch.float16):
        raise NotImplementedError


def _cond(cfg, B, g, size, last_uc, last_c):
    """(uc, c, added_cond_kwargs) with 2B added rows: time ids (size, size, 0, 0, last) per row, `last` the target size
    for the base (6 ids) or the aesthetic score for the refiner (5 ids)."""
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().to(dev)
    row = lambda last: [size, size, 0., 0.] + list(last)  # noqa: E731
    tids = torch.tensor([row(last_uc)] * B + [row(last_c)] * B, dtype=torch.float16).to(dev)
    assert tids.shape[1] == cfg.num_time_ids
    return uc, c, {"text_embeds": pooled, "time_ids": tids}


def _base_cond(cfg, B, g, size):
    return _cond(cfg, B, g, size, (size, size), (size, size))


def _refiner_cond(cfg, B, g, size):
    return _cond(cfg, B, g, size, (2.5,), (6.0,))


def _bind(net, B, hw, cond):
    uc, c, add = cond
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())


# ---- the add-embedding ------------------------------------------------------------------------------------------

def test_time_id_geometry_refused():
    """The handle derives n_time_ids = (projection_class_embeddings_input_dim - pooled_dim) / addition_time_embed_dim
    and refuses a count that is not whole or not in 1..8 when it is created (an input check)."""
    from cfgpp_b200 import _native as nv, config as C
    from cfgpp_b200.engine import NativeUNet
    base = C.tiny_sdxl_refiner_config()  # pooled 64, 32 per id
    for ain, msg in ((64 + 5 * 32 + 16, "whole multiple of addition_time_embed_dim"),
                     (64 + 9 * 32, "1..8 time ids"), (64, "whole multiple")):
        cfg = dataclasses.replace(base, projection_class_embeddings_input_dim=ain)
        with pytest.raises(nv.NativeError, match=msg) as e:
            NativeUNet(cfg, {}, dev)
        print(f"[refiner] projection_class_embeddings_input_dim {ain}: refused: {e.value}")


def test_tiny_refiner_forward_vs_oracle():
    """The 5-id add-embedding (1 + 5 launches) and the refiner topology at test widths against the oracle."""
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg = C.tiny_sdxl_refiner_config()
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    g = torch.Generator().manual_seed(3)
    B, hw = 2, 32
    z = torch.randn(B, 4, hw, hw, generator=g).to(dev)
    cond = _refiner_cond(cfg, B, g, 256.)
    net = NativeUNet(cfg, sd, dev)
    _bind(net, B, hw, cond)
    eu, ec = net.predict_noise(z, 301.0)
    prompt_launches = net.plan_stats["prompt_launches"]
    net.close()
    uc, c, add = cond
    r = OracleCudaUNet(cfg, sd, dev)(torch.cat([z] * 2), torch.tensor(301, device=dev), torch.cat([uc, c]), add)["sample"]
    e = rel_l2(torch.cat([eu, ec]), r)
    # the time ids matter: the aesthetic score changes the output
    add2 = {"text_embeds": add["text_embeds"], "time_ids": add["time_ids"].clone()}
    add2["time_ids"][:, 4] = 9.0
    r2 = OracleCudaUNet(cfg, sd, dev)(torch.cat([z] * 2), torch.tensor(301, device=dev), torch.cat([uc, c]), add2)["sample"]
    print(f"[refiner] tiny refiner UNet B={B} {hw}x{hw}: rel-L2 vs fp16 oracle {e:.3e} "
          f"(other aesthetic score: {rel_l2(r2, r):.3e}); {prompt_launches} prompt launches")
    assert e <= 5e-3 and rel_l2(r2, r) > 10 * e


@pytest.mark.parametrize("B,h,w,t", [(1, 128, 128, 181), (2, 128, 128, 41), (1, 152, 104, 121)])
def test_refiner_unet_full_geometry(B, h, w, t):
    """The real refiner UNet (2.26 B params, 384-wide level 0 without attention, 24 x 64 heads at 1536 channels,
    context 1280) at 1024^2 and at the 1216 x 832 bucket, synthetic weights."""
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    from oracle import unet as O
    cfg = C.sdxl_refiner_config()
    sd = Wt.synthetic_state_dict(cfg, seed=77, device=dev)
    g = torch.Generator().manual_seed(B + h + w)
    z = torch.randn(B, 4, h, w, generator=g).to(dev)
    uc, c, add = _refiner_cond(cfg, B, g, 8. * h)
    net = NativeUNet(cfg, sd, dev)
    net.prepare(B, h, w)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
    eu, ec = net.predict_noise(z, float(t))
    got = torch.cat([eu, ec]).float()
    ws = net.workspace_bytes
    net.close()
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
    ref16 = OracleCudaUNet(cfg, sd, dev)
    r16 = ref16(z_in, t_in, ctx, add)["sample"].float()
    del ref16
    m32 = O.build_unet(oracle_cfg(cfg), sd, dtype=torch.float32, device=dev)
    with torch.no_grad():
        r32 = m32(z_in, t_in, ctx.float(), {k: v.float() for k, v in add.items()})["sample"]
    del m32
    e16, e32, o32 = rel_l2(got, r16), rel_l2(got, r32), rel_l2(r16, r32)
    print(f"[refiner] UNet B={B} latent {h}x{w} t={t}: rel-L2 vs fp16 oracle {e16:.3e}, vs fp32 {e32:.3e} "
          f"(fp16 oracle vs fp32 {o32:.3e}); workspace {ws / 2**30:.2f} GiB")
    assert torch.isfinite(got).all() and e16 <= 5e-3 and e32 <= 1.5 * o32 + 1e-4


# ---- split trajectories at real widths --------------------------------------------------------------------------------

def _release_gpu_memory():
    """Hand this process's device memory back: cached engines, then PyTorch's caching allocator."""
    from cfgpp_b200 import latent_sdxl as LX
    LX.release_engines()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture
def real_experts():
    """Native engines and fp16 oracles of the real base and refiner (about 25 GB of device memory with their
    workspaces): built per test and released right after it, so nothing of them outlives the test that uses them."""
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    B, hw = 2, 128
    g = torch.Generator().manual_seed(17)
    out = {"B": B, "hw": hw, "z": torch.randn(B, 4, hw, hw, generator=g).to(dev)}
    for name, cfg, seed, mk in (("base", C.sdxl_config(), 1234, _base_cond),
                                ("refiner", C.sdxl_refiner_config(), 4321, _refiner_cond)):
        sd = Wt.synthetic_state_dict(cfg, seed=seed, device=dev)
        out[name] = (NativeUNet(cfg, sd, dev), OracleCudaUNet(cfg, sd, dev), mk(cfg, B, g, 1024.))
        del sd
    yield out
    for name in ("base", "refiner"):
        out[name][0].close()
    out.clear()
    _release_gpu_memory()


@pytest.mark.parametrize("method,nfe", [("ddim_cfg++", 50), ("dpm++_2m_cfgpp", 25)])
def test_split_trajectory_vs_oracle_1024(real_experts, method, nfe):
    """Base steps [0, k) then refiner steps [k, n) at 1024^2, B = 2, lambda 0.6, denoising_end 0.8: teacher-forced per
    step (eps of both halves, and z_{t-1} for DDIM) and the free-running fused trajectory with the hand-off."""
    from cfgpp_b200 import schedule as S
    from oracle import schedule as OS, sdxl_refiner as OR
    B, hw, z, lam = real_experts["B"], real_experts["hw"], real_experts["z"], 0.6
    (nb, ob, cb), (nr, orf, cr) = real_experts["base"], real_experts["refiner"]
    tb, sch = OS.make_tables(nfe), S.Schedule.make(nfe)
    rec = []
    if method == "ddim_cfg++":
        k = S.expert_split(sch.timesteps, 0.8, nfe)
        ref = OR.sdxl_ddim_cfgpp_split(ob, orf, tb, z, cb, cr, lam, k, record=rec)
        steps = S.ddim_cfgpp_steps(sch, lam, sdxl_indexing=True)
        mode, dt, x0, which = S.STEP_DDIM_CFGPP, torch.float32, z, 1
    else:
        k = S.expert_split(sch.timesteps, 0.8, nfe - 1)
        ref = OR.sdxl_dpmpp_2m_cfgpp_split(ob, orf, tb, z, cb, cr, lam, k, record=rec)
        steps, sigma0 = S.dpmpp_2m_cfgpp_steps(sch, lam, restart_at=k)
        mode, dt, x0, which = S.STEP_DPMPP2M_CFGPP, torch.float16, z.half() * sigma0, 0
    key = "zt" if which == 1 else "x"
    assert len(rec) == len(steps) and torch.equal(rec[0][key], x0)
    for net, cond in ((nb, cb), (nr, cr)):
        _bind(net, B, hw, cond)
        net.set_schedule(mode, dt, steps)
    worst = 0.0
    for i, r in enumerate(rec):
        net = nb if i < k else nr
        eu, ec = net.predict_noise(r[key], steps[i].t, steps[i].in_scale)
        errs = [rel_l2(eu, r["noise_uc"]), rel_l2(ec, r["noise_c"])]
        if which == 1:
            net.set_state(r[key])
            net.run_steps(i, 1)
            if i + 1 < len(rec):
                errs.append(rel_l2(net.get_state(0), rec[i + 1][key]))
        worst = max(worst, *errs)
        assert max(errs) <= 5e-3, f"{method} step {i} ({'base' if i < k else 'refiner'}): {errs}"
    nb.set_state(x0)
    nb.run_steps(0, k)
    nr.set_state(nb.get_state(0))
    nr.run_steps(k, len(steps) - k)
    e = rel_l2(nr.get_state(which), ref)
    print(f"[refiner] split {method} NFE={nfe} 1024^2 B={B}: base {k} + refiner {len(steps) - k} steps, teacher-forced "
          f"worst {worst:.3e}, free-running final {'z0t' if which else 'x'} {e:.3e}")
    assert e <= 3e-2


# ---- plumbing: same weights, fused == callback, batching ---------------------------------------------------------------

@pytest.fixture(scope="module")
def tiny():
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.conditioning import SyntheticTextEncoder
    base, ref = C.tiny_sdxl_config(), C.tiny_sdxl_refiner_config()
    return {"base": (base, Wt.synthetic_state_dict(base, seed=1234, device=dev)),
            "refiner": (ref, Wt.synthetic_state_dict(ref, seed=99, device=dev)),
            "text": (SyntheticTextEncoder(64, 0), SyntheticTextEncoder(64, 64))}


def _solver(method, tiny, nfe, vae=None, text=True):
    from cfgpp_b200 import latent_sdxl as LX
    cfg, sd = tiny["base"]
    kw = {"text_encoders": tiny["text"]} if text else {}
    return LX.get_solver(method, solver_config=SimpleNamespace(num_sampling=nfe), device=dev, unet_config=cfg,
                         state_dict=sd, vae=vae or LatentVAE(), **kw)


@pytest.mark.parametrize("method", ["ddim_cfg++", "ddim"])
def test_same_weights_refiner_is_unsplit(tiny, method):
    """A 'refiner' engine built from the base's config and weights, under the base's own conditioning: the split fused
    trajectory is bit-identical to the unsplit one (the hand-off copies the state exactly and changes nothing else)."""
    from cfgpp_b200 import latent_sdxl as LX
    cfg, sd = tiny["base"]
    s = _solver(method, tiny, 10)
    twin = LX.SDXLRefiner(model_key="same-weights-twin", device=dev, unet_config=cfg, state_dict=sd)
    assert twin.unet is not s.unet
    g = torch.Generator().manual_seed(5)
    B = 2
    zT = torch.randn(B, 4, 32, 32, generator=g)
    uc, c, add = _base_cond(cfg, B, g, 256.)
    lam = [0.6, 0.9]
    ref = s.reverse_process(uc, c, lam, add, (256, 256), None, zT=zT)
    got = s.reverse_process(uc, c, lam, add, (256, 256), None, zT=zT, refiner=twin, refiner_cond=(uc, c, add),
                            denoising_end=0.8)
    print(f"[refiner] {method} same-weights split (k = 8 of 10) vs unsplit: bit-identical {torch.equal(got, ref)}")
    assert torch.equal(got, ref)


@pytest.mark.parametrize("method", ["ddim_cfg++", "ddim", "dpm++_2m_cfgpp"])
def test_fused_equals_callback_across_hand_off(tiny, method):
    from cfgpp_b200 import latent_sdxl as LX
    s = _solver(method, tiny, 10)
    rcfg, rsd = tiny["refiner"]
    refiner = LX.SDXLRefiner(model_key="synthetic:99", device=dev, unet_config=rcfg, state_dict=rsd)
    g = torch.Generator().manual_seed(6)
    B = 2
    zT = torch.randn(B, 4, 32, 32, generator=g)
    cb_, rc = _base_cond(s.cfg, B, g, 256.), _refiner_cond(rcfg, B, g, 256.)
    lam = [0.4, 0.8]
    seen = []
    outs = []
    for callback in (None, lambda i, t, kw: seen.append(i) or kw):
        outs.append(s.reverse_process(*cb_[:2], lam, cb_[2], (256, 256), callback, zT=zT, refiner=refiner,
                                      refiner_cond=rc, denoising_end=0.8))
    n = 10 if method != "dpm++_2m_cfgpp" else 9
    unsplit = s.reverse_process(*cb_[:2], lam, cb_[2], (256, 256), None, zT=zT)
    print(f"[refiner] {method}: fused == callback across the hand-off {torch.equal(*outs)} (callback steps {seen}); "
          f"split vs base-only rel-L2 {rel_l2(outs[0], unsplit):.3e}")
    assert seen == list(range(n)) and torch.equal(outs[0], outs[1])
    assert not torch.equal(outs[0], unsplit)


def test_sample_with_refiner_batch_equals_serial(tiny):
    """sample() with a refiner at B = 2 and guidance [0.6, 1.0]: image i equals the B = 1 call (conditioning of both
    experts from the prompts through the native tiny CLIP towers; the refiner reuses the base's second tower)."""
    from cfgpp_b200 import latent_sdxl as LX
    vae = LatentVAE()
    s = _solver("ddim_cfg++", tiny, 6, vae=vae, text=False)
    rcfg, rsd = tiny["refiner"]
    refiner = LX.SDXLRefiner(model_key="synthetic:99", device=dev, unet_config=rcfg, state_dict=rsd)
    zT = torch.randn(2, 4, 32, 32, generator=torch.Generator().manual_seed(8))
    prompts, lams = ["a lighthouse at dusk", "a bowl of fruit"], [0.6, 1.0]
    run = lambda p, lam, z: s.sample(prompt1=["", p], prompt2=["", p], cfg_guidance=lam, target_size=(256, 256),  # noqa: E731
                                     zT=z, refiner=refiner, denoising_end=0.8)
    img = run(prompts, lams, zT)
    assert img.shape == (2, 3, 256, 256) and len(vae.latents) == 1  # decoded once, after the refiner
    lat = vae.latents[-1]
    s.sample(prompt1=["", prompts], prompt2=["", prompts], cfg_guidance=lams, target_size=(256, 256), zT=zT)
    base_only = vae.latents[-1]
    errs = []
    for b in range(2):
        run(prompts[b], lams[b], zT[b:b + 1])
        errs.append(rel_l2(lat[b:b + 1], vae.latents[-1]))
    print(f"[refiner] sample() B=2 lambda {lams}: batch vs serial final-latent rel-L2 "
          + ", ".join(f"{e:.3e}" for e in errs) + f"; refined vs base-only {rel_l2(lat, base_only):.3e}")
    assert max(errs) <= 3e-2 and not torch.equal(lat, base_only)


@pytest.mark.parametrize("method", ["euler_cfg++", "ddim_cfg++_lightning"])
def test_refiner_rejected(tiny, method):
    from cfgpp_b200 import latent_sdxl as LX
    s = _solver(method, tiny, 4)
    with pytest.raises(ValueError, match="dpm\\+\\+_2m_cfgpp") as e:
        s.sample(prompt1=["", "a"], prompt2=["", "a"], cfg_guidance=1.0, refiner=SimpleNamespace())
    print(f"[refiner] {method} with a refiner: {e.value}")


# ---- end to end -------------------------------------------------------------------------------------------------------

def test_text_to_img_example_with_refiner(tmp_path):
    """`python -m examples.text_to_img --model sdxl --denoising_end 0.8`: real-width base and refiner on synthetic
    weights, CLIP-L + bigG and the SDXL VAE, 1024^2. The example is a second process that needs both real UNets on the
    device, so this process first gives back whatever earlier tests left cached."""
    _release_gpu_memory()
    free, total = torch.cuda.mem_get_info()
    print(f"[refiner] device memory free before the example: {free / 2**30:.1f} of {total / 2**30:.1f} GiB")
    out = subprocess.run([sys.executable, "-m", "examples.text_to_img", "--model", "sdxl", "--denoising_end", "0.8",
                          "--NFE", "5", "--cfg_guidance", "0.6", "--prompt", "a cat", "--workdir", str(tmp_path)],
                         cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    img = torch.load(tmp_path / "result" / "generated.pt")
    print(f"[refiner] examples.text_to_img --model sdxl --denoising_end 0.8: {tuple(img.shape)}, "
          f"finite {bool(torch.isfinite(img).all())}")
    assert img.shape == (1, 3, 1024, 1024) and torch.isfinite(img).all()
    assert "synthetic" in out.stderr
