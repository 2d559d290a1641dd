"""Batched sampling with a per-image guidance scale: the step kernel's guidance table (bitwise against the scalar step
per row, every step mode and second_order bit, fp16 and fp32 state), fused vs callback trajectories, batch vs serial
`sample()` for every deterministic text-to-image method, and batched trajectories against the oracle.

Tolerances: step kernel and fused-vs-callback DDIM bit-identical; batch vs serial final latent rel-L2 <= 3e-2 (the
free-running bound of DESIGN §3: a batch runs other GEMM shapes, so rows differ in the last bits and the trajectory
amplifies that); teacher-forced per-step rel-L2 <= 5e-3 against the oracle."""
from types import SimpleNamespace

import pytest
import torch

from helpers import build_pair, coef_variants, make_inputs, rel_l2

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


class RowLambda:
    """A per-row guidance scale for the oracle loops: `lam * t` multiplies row b of t by the Python float lam[b], the
    op the reference's loop runs for a single image with that scalar."""
    def __init__(self, lams):
        self.lams = [float(v) for v in lams]

    def __mul__(self, t):
        return torch.cat([v * t[b:b + 1] for b, v in enumerate(self.lams)])

    __rmul__ = __mul__


class LatentVAE:
    """Stand-in VAE that keeps the latent it is asked to decode (the tests compare final latents)."""
    def __init__(self):
        self.latents = []

    def decode(self, z):
        self.latents.append(z.detach().clone())
        return torch.zeros(z.shape[0], 3, 8 * z.shape[2], 8 * z.shape[3], device=z.device)

    def encode(self, x, dtype=torch.float16):
        raise NotImplementedError


# ---- 1. step kernel: the guidance table reaches every mode and bit, bitwise ---------------------------------------

def test_step_kernel_guidance_table_bitwise_per_row():
    from cfgpp_b200 import _native as nv
    lams = [0.0, 0.6, 1.0, 7.5]
    shape = (len(lams), 4, 16, 24)
    g = torch.Generator().manual_seed(0)
    lam_dev = torch.tensor(lams, dtype=torch.float32, device=dev)
    for k, (method, dt, coef, uses_aux, slots) in enumerate(coef_variants()):
        eu = torch.randn(shape, generator=g).half().to(dev)
        ec = torch.randn(shape, generator=g).half().to(dev)
        z0 = (torch.randn(shape, generator=g) * 3).to(dt).to(dev)
        aux0 = torch.randn(shape, generator=g).to(dt).to(dev) if uses_aux else None
        noise = torch.randn(max(slots, 1), *shape, generator=g).half().to(dev) if slots else None
        z = z0.clone()
        aux = aux0.clone() if uses_aux else None
        zt = nv.op_cfgpp_step(eu, ec, method, coef, z, aux=aux, noise=noise, lambdas=lam_dev)
        tag = f"variant {k}: method {method} {dt} second_order {coef.second_order}"
        for b, lam in enumerate(lams):
            c1 = type(coef).from_buffer_copy(coef)
            c1.lambda_ = lam
            zb = z0[b:b + 1].clone()
            ab = aux0[b:b + 1].clone() if uses_aux else None
            nb = noise[:, b:b + 1].contiguous() if slots else None
            ztb = nv.op_cfgpp_step(eu[b:b + 1].contiguous(), ec[b:b + 1].contiguous(), method, c1, zb, ab, noise=nb)
            assert torch.equal(z[b:b + 1], zb) and torch.equal(zt[b:b + 1], ztb), f"{tag} row {b}"
            if uses_aux:
                assert torch.equal(aux[b:b + 1], ab), f"{tag} row {b} aux"


# ---- 2. engine: the table reaches the fused graph and apply_step, and clearing it restores the scalar ------------

def test_engine_guidance_table_fused_unfused_and_clear():
    from cfgpp_b200 import schedule as S
    cfg, sd, net, _ = build_pair("tiny_sdxl", dev)
    B, hw, lams = 3, 32, [0.0, 0.6, 1.0]
    z, uc, c, add = make_inputs(cfg, B, hw, dev)
    steps = S.ddim_cfgpp_steps(S.Schedule.make(5), 0.6, True)
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())

    def fused(guidance):
        net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps, guidance)
        net.set_state(z)
        net.run_steps(0, len(steps))
        return net.get_state(0).clone(), net.get_state(1).clone()

    scalar = fused(None)
    guided = fused(lams)
    assert not torch.equal(scalar[0], guided[0])
    assert torch.equal(fused(None)[0], scalar[0])          # cleared: the scalar results, bit for bit
    assert torch.equal(fused(lams)[0], guided[0])          # set again on the same captured graph
    # un-fused seam (callback path): predict_noise + apply_step with the table set
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps, lams)
    net.set_state(z)
    for i, st in enumerate(steps):
        eu, ec = net.predict_noise(net.get_state(0), st.t)
        net.apply_step(i, eu, ec)
    assert torch.equal(net.get_state(0), guided[0]) and torch.equal(net.get_state(1), guided[1])
    # a lambda of 0.6 in the table is the scalar 0.6 for that image
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps, [0.6] * B)
    net.set_state(z)
    net.run_steps(0, len(steps))
    assert torch.equal(net.get_state(0), scalar[0])
    with pytest.raises(ValueError):
        net.set_guidance([0.5, 0.5])
    net.close()


# ---- 3. fused == callback with a per-image lambda ---------------------------------------------------------------

def test_fused_equals_callback_with_per_image_guidance_ddim():
    from cfgpp_b200 import latent_diffusion as LD
    cfg, sd, net, _ = build_pair("tiny_sd15", dev)
    net.close()
    z, uc, c, _ = make_inputs(cfg, 3, 32, dev)
    s = LD.get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=5), device=dev, unet_config=cfg,
                      state_dict=sd, vae=LatentVAE())
    lams = [0.0, 0.6, 1.0]
    fused = s.reverse_process(uc, c, lams, z)
    seen = []
    cb = s.reverse_process(uc, c, lams, z, callback_fn=lambda i, t, kw: (seen.append(i), kw)[1])
    assert seen == list(range(5)) and torch.equal(fused, cb)


@pytest.mark.parametrize("method", ["dpm++_2m_cfg++", "euler_a_cfg++"])
def test_fused_equals_callback_with_per_image_guidance_kdiffusion(method):
    """The k-diffusion callback path runs the update as torch ops, the per-image mix row by row with Python floats;
    the fused kernel rounds at the same points, so the two trajectories are bit-identical."""
    from cfgpp_b200 import latent_diffusion as LD
    cfg, sd, net, _ = build_pair("tiny_sd15", dev)
    net.close()
    z, uc, c, _ = make_inputs(cfg, 3, 32, dev)
    s = LD.get_solver(method, solver_config=SimpleNamespace(num_sampling=6), device=dev, unet_config=cfg,
                      state_dict=sd, vae=LatentVAE())
    lams = [0.0, 0.6, 1.0]
    x0 = (z * (s.karras_sigmas()[0] ** 2 + 1) ** 0.5).half()
    torch.manual_seed(77)
    d_cb, x_cb = s.reverse_process(uc, c, lams, x0.clone(), callback_fn=lambda i, t, kw: kw)
    torch.manual_seed(77)
    d_f, x_f = s.reverse_process(uc, c, lams, x0.clone())
    for b in range(3):
        e_x, e_d = rel_l2(x_f[b], x_cb[b]), rel_l2(d_f[b], d_cb[b])
        print(f"{method} image {b} (lambda {lams[b]}): fused vs callback x {e_x:.3e}, denoised {e_d:.3e}")
    assert torch.equal(x_f, x_cb) and torch.equal(d_f, d_cb)
    # the per-image lambda really acts per image: image 0 (lambda 0) ignores its prompt
    torch.manual_seed(77)
    _, x_other = s.reverse_process(uc, c.roll(1, 0), lams, x0.clone())
    assert rel_l2(x_other[0], x_f[0]) < 2e-3 and rel_l2(x_other[1], x_f[1]) > 1e-2


# ---- 4. batch == serial for every deterministic text-to-image method ---------------------------------------------

SD15_METHODS = ["ddim", "ddim_cfg++", "euler", "euler_cfg++", "dpm++_2m", "dpm++_2m_cfg++"]
SDXL_METHODS = ["ddim", "euler", "ddim_cfg++", "dpm++_2m_cfgpp", "euler_cfg++", "ddim_lightning", "euler_lightning",
                "ddim_cfg++_lightning", "dpm++_2m_cfgpp_lightning", "euler_cfg++_lightning"]


@pytest.fixture(scope="module")
def tiny_weights():
    from cfgpp_b200 import config as C, weights as Wt
    return {name: (C.CONFIGS[name](), Wt.synthetic_state_dict(C.CONFIGS[name](), seed=1234, device=dev))
            for name in ("tiny_sd15", "tiny_sdxl")}


def _batch_vs_serial(solver, vae, run, lams, prompts, zT, tag):
    batch_img = run(prompts, lams, zT)
    assert batch_img.shape[0] == len(prompts)
    lat_batch = vae.latents[-1]
    errs = []
    for b in range(len(prompts)):
        img_b = run(prompts[b], lams[b], zT[b:b + 1])
        assert img_b.shape == batch_img[b:b + 1].shape
        errs.append(rel_l2(lat_batch[b:b + 1], vae.latents[-1]))
    print(f"{tag}: batch vs serial final-latent rel-L2 per image = " + ", ".join(f"{e:.3e}" for e in errs))
    assert max(errs) <= 3e-2, tag


@pytest.mark.parametrize("method", SD15_METHODS)
def test_batch_equals_serial_sd15(method, tiny_weights):
    from cfgpp_b200 import latent_diffusion as LD
    cfg, sd = tiny_weights["tiny_sd15"]
    vae = LatentVAE()
    s = LD.get_solver(method, solver_config=SimpleNamespace(num_sampling=5), device=dev, unet_config=cfg,
                      state_dict=sd, vae=vae)
    zT = torch.randn(3, 4, cfg.sample_size, cfg.sample_size, generator=torch.Generator().manual_seed(3))
    run = lambda p, lam, z: s.sample(cfg_guidance=lam, prompt=["", p], zT=z)  # noqa: E731
    _batch_vs_serial(s, vae, run, [0.0, 0.6, 1.0], ["a red cube", "a dog on grass", "city at night"], zT,
                     f"sd15 {method}")


@pytest.mark.parametrize("method", SDXL_METHODS)
def test_batch_equals_serial_sdxl(method, tiny_weights):
    from cfgpp_b200 import latent_sdxl as LX
    cfg, sd = tiny_weights["tiny_sdxl"]
    vae = LatentVAE()
    kw = dict(solver_config=SimpleNamespace(num_sampling=4 if "lightning" in method else 5), device=dev,
              unet_config=cfg, state_dict=sd, vae=vae)
    s = LX.get_solver(method, **kw)
    hw = cfg.sample_size
    zT = torch.randn(3, 4, hw, hw, generator=torch.Generator().manual_seed(4))
    lams = [1.0, 1.0, 1.0] if "lightning" in method else [0.0, 0.6, 1.0]
    run = lambda p, lam, z: s.sample(prompt1=["", p], prompt2=["", p], cfg_guidance=lam,  # noqa: E731
                                     target_size=(8 * hw, 8 * hw), zT=z)
    _batch_vs_serial(s, vae, run, lams, ["a red cube", "a dog on grass", "city at night"], zT, f"sdxl {method}")


def test_batch_without_zT_draws_each_image_in_order(tiny_weights):
    from cfgpp_b200 import latent_sdxl as LX
    from cfgpp_b200.utils.log_util import set_seed
    cfg, sd = tiny_weights["tiny_sdxl"]
    vae = LatentVAE()
    s = LX.get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=4), device=dev, unet_config=cfg,
                      state_dict=sd, vae=vae)
    hw, prompts, lams = cfg.sample_size, ["one", "two"], [0.4, 0.8]
    set_seed(11)
    img = s.sample(prompt1=["", prompts], prompt2=["", prompts], cfg_guidance=lams, target_size=(8 * hw, 8 * hw))
    assert img.shape == (2, 3, 8 * hw, 8 * hw)
    lat = vae.latents[-1]
    set_seed(11)
    for b in range(2):
        s.sample(prompt1=["", prompts[b]], prompt2=["", prompts[b]], cfg_guidance=lams[b],
                 target_size=(8 * hw, 8 * hw))
        e = rel_l2(lat[b:b + 1], vae.latents[-1])
        print(f"sdxl ddim_cfg++ without zT, image {b}: batch vs serial rel-L2 {e:.3e}")
        assert e <= 3e-2


def test_batch_equals_serial_sdxl_1024():
    """Full-size SDXL UNet (synthetic weights) at 1024^2, B = 2, lambda = (0.4, 0.8), 3 DDIM CFG++ steps."""
    from cfgpp_b200 import latent_sdxl as LX
    from cfgpp_b200.conditioning import SyntheticTextEncoder
    vae = LatentVAE()
    s = LX.get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=3), device=dev, model_key="synthetic:5",
                      text_encoders=(SyntheticTextEncoder(768, 0), SyntheticTextEncoder(1280, 1280)), vae=vae)
    zT = torch.randn(2, 4, 128, 128, generator=torch.Generator().manual_seed(6))
    run = lambda p, lam, z: s.sample(prompt1=["", p], prompt2=["", p], cfg_guidance=lam, zT=z)  # noqa: E731
    try:
        _batch_vs_serial(s, vae, run, [0.4, 0.8], ["a lighthouse at dusk", "a bowl of fruit"], zT, "sdxl 1024 ddim_cfg++")
    finally:
        LX.release_engines()


# ---- 5. against the oracle ---------------------------------------------------------------------------------------

def test_teacher_forced_batched_ddim_vs_oracle():
    from cfgpp_b200 import batching as Bt, schedule as S
    from oracle import samplers as OSm, schedule as OS
    cfg, sd, net, ref = build_pair("tiny_sdxl", dev)
    B, hw, nfe, lams = 3, 32, 8, [0.0, 0.6, 1.0]
    z, uc, c, add = make_inputs(cfg, B, hw, dev)
    pooled_neg, pooled_pos = add["text_embeds"][:B], add["text_embeds"][B:]
    te, ti = Bt.sdxl_added_conditions(pooled_neg, pooled_pos, add["time_ids"][:1], add["time_ids"][:1], lams, B)
    add = {"text_embeds": te, "time_ids": ti.to(dev)}
    tb = OS.make_tables(nfe)
    rec = []
    z0_ref = OSm.sdxl_ddim_cfgpp(ref, tb, z, uc, c, RowLambda(lams), add, record=rec)
    steps = S.ddim_cfgpp_steps(S.Schedule.make(nfe), lams, sdxl_indexing=True)
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps, lams)
    worst = 0.0
    for i, r in enumerate(rec):
        net.set_state(r["zt"])
        net.run_steps(i, 1)
        if i + 1 < len(rec):
            worst = max(worst, max(rel_l2(net.get_state(0)[b], rec[i + 1]["zt"][b]) for b in range(B)))
    print(f"teacher-forced batched ddim_cfg++ (lambda {lams}): worst per-image per-step rel-L2 {worst:.3e}")
    assert worst <= 5e-3
    net.set_state(z)
    net.run_steps(0, nfe)
    e = [rel_l2(net.get_state(1)[b], z0_ref[b]) for b in range(B)]
    print("free-running per image: " + ", ".join(f"{v:.3e}" for v in e))
    assert max(e) <= 3e-2
    net.close()


def test_teacher_forced_batched_dpmpp_vs_oracle():
    from cfgpp_b200 import schedule as S
    from oracle import samplers as OSm, schedule as OS
    cfg, sd, net, ref = build_pair("tiny_sdxl", dev)
    B, hw, nfe, lams = 3, 32, 8, [0.3, 0.6, 0.9]
    z, uc, c, add = make_inputs(cfg, B, hw, dev)
    tb = OS.make_tables(nfe)
    rec = []
    x_ref = OSm.sdxl_dpmpp_2m_cfgpp(ref, tb, z, uc, c, RowLambda(lams), add, record=rec)
    steps, sigma0 = S.dpmpp_2m_cfgpp_steps(S.Schedule.make(nfe), lams)
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
    net.set_schedule(S.STEP_DPMPP2M_CFGPP, torch.float16, steps, lams)
    # teacher-forced first (Euler-form) step; the 2M steps also read the previous estimate the engine keeps in aux
    net.set_state(rec[0]["x"])
    net.run_steps(0, 1)
    e0 = max(rel_l2(net.get_state(0)[b], rec[1]["x"][b]) for b in range(B))
    net.set_state(z.to(torch.float16) * sigma0)
    net.run_steps(0, len(steps))
    e = [rel_l2(net.get_state(0)[b], x_ref[b]) for b in range(B)]
    print(f"batched dpm++_2m_cfgpp (lambda {lams}): teacher-forced step 0 rel-L2 {e0:.3e}, free-running per image "
          + ", ".join(f"{v:.3e}" for v in e))
    assert e0 <= 5e-3 and max(e) <= 3e-2
    net.close()


@pytest.mark.parametrize("method", ["euler_a_cfg++", "dpm++_2s_a_cfg++"])
def test_batched_ancestral_vs_oracle_same_noise(method):
    from cfgpp_b200 import latent_diffusion as LD
    from oracle import samplers as OSm, schedule as OS
    cfg, sd, net, ref = build_pair("tiny_sd15", dev)
    net.close()
    nfe, lams, hw = 6, [0.0, 0.6, 1.0], 32
    z, uc, c, _ = make_inputs(cfg, 3, hw, dev)
    s = LD.get_solver(method, solver_config=SimpleNamespace(num_sampling=nfe), device=dev, unet_config=cfg,
                      state_dict=sd, vae=LatentVAE())
    tb = OS.make_tables(nfe)
    sigmas = s.karras_sigmas()
    x0 = OSm.kd_start_state(z, sigmas)
    lam = RowLambda(lams)
    oracle = {"euler_a_cfg++": lambda: OSm.kd_euler_cfgpp(ref, tb, x0.clone(), sigmas, uc, c, lam, ancestral=True),
              "dpm++_2s_a_cfg++": lambda: OSm.kd_dpmpp_2s_a_cfgpp(ref, tb, x0.clone(), sigmas, uc, c, lam)}[method]
    torch.manual_seed(123)
    d_ref, x_ref = oracle()
    torch.manual_seed(123)
    d, x = s.reverse_process(uc, c, lams, x0.clone())
    e = [rel_l2(x[b], x_ref[b]) for b in range(3)]
    print(f"batched {method} vs oracle (same batch noise), final x per image: " + ", ".join(f"{v:.3e}" for v in e))
    assert max(e) <= 3e-2 and rel_l2(d, d_ref) <= 3e-2
