"""Stable Diffusion 2.x on the GPU: the v -> eps conversion of the fused step kernel (bit-exact against its torch
restatement and against convert-then-step), the epsilon path of a handle that carries prediction_type = 0 (bit-identical
to a handle created without the field), the SD 2 UNet at 768^2 / 512^2 / 768x512 against the oracle, `ddim_cfg++` with
v-prediction against the oracle's v rule, fused == callback trajectories, the ViT-H text tower against transformers,
and `sample()` / `examples.inversion --model sd20` end to end. Every test prints what it measured (`pytest -s`).

Stated tolerances: UNet rel-L2 <= 5e-3 against the fp16-autocast oracle and an fp32 error <= 1.5x the fp16 oracle's
own (DESIGN section 3); teacher-forced step <= 5e-3, free-running final latent <= 3e-2; text tower <= 5e-3."""
import math
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from helpers import OracleCudaUNet, coef_variants, oracle_cfg, rel_l2

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
ROOT = Path(__file__).resolve().parent.parent


def _model_input(z, scale):
    """conv_in's UNet input: fp16 arithmetic for an fp16 state, an fp32 product cast to fp16 for an fp32 one."""
    if scale is None:
        return z.half()
    if z.dtype == torch.float16:
        return (z.float() * scale).half()
    return (z * torch.tensor(scale, dtype=torch.float32)).half()


def _v_to_eps_ref(v, z, a, b, scale):
    x_in = _model_input(z, scale)
    return (v.float() * a + x_in.float() * b).half()


# ---- the conversion ---------------------------------------------------------------------------------------------

def test_v_to_eps_bit_exact():
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(1)
    n = 1 << 16
    v_rand = (torch.randn(n, generator=g) * 2).half()
    # adversarial: |v| up to the fp16 maximum (fp32 sums that leave the fp16 range), fp16 subnormal v and x_in, exact
    # ties, signed zeros
    big = torch.tensor([65504., -65504., 60000., 32768., 1e4, -1e4], dtype=torch.float16)
    sub = torch.tensor([6e-8, -6e-8, 1.2e-7, 3e-6, 6.1e-5, -6.1e-5, 0.0, -0.0], dtype=torch.float16)
    v_adv = torch.cat([big, sub, big.flip(0), sub.flip(0)]).repeat(n // 28 + 1)[:n]
    z_rand = torch.randn(n, generator=g) * 3
    z_adv = torch.cat([sub.float(), big.float(), sub.float().flip(0) * 3, big.float().flip(0)]).repeat(n // 28 + 1)[:n]
    c_in = 1.0 / math.sqrt(14.6146 ** 2 + 1)
    levels = [(0.9995749, 0.0291551), (0.0682, 0.99767), (c_in, 14.6146 * c_in), (1.0, 0.0)]
    checked = 0
    for v, z in ((v_rand, z_rand), (v_adv, z_adv), (v_adv, z_rand), (v_rand, z_adv)):
        for zt in (z.half(), z.float()):
            for scale in (None, c_in):
                sdev = torch.tensor([scale], dtype=torch.float32, device=dev) if scale is not None else None
                for a, b in levels:
                    a, b = float(torch.tensor(a, dtype=torch.float32)), float(torch.tensor(b, dtype=torch.float32))
                    got = nv.op_v_to_eps(v.to(dev), zt.to(dev), a, b, in_scale=sdev)
                    ref = _v_to_eps_ref(v.to(dev), zt.to(dev), a, b, scale)
                    assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), \
                        f"v_to_eps {zt.dtype} scale {scale} (a, b) = ({a}, {b})"
                    checked += 1
    print(f"[sd2] cfgpp_op_v_to_eps: {checked} cases x {n} elements bit-exact against the fp32 torch restatement")


@pytest.mark.parametrize("B,H,W", [(1, 17, 12), (3, 12, 8)])
def test_conv_out_step_v_equals_convert_then_step(B, H, W):
    """The v launch writes the raw v and then steps exactly as cfgpp_op_v_to_eps followed by the standalone step on that
    v would: every step mode and second_order bit, scalar and per-image guidance, with and without the noise table."""
    from cfgpp_b200 import _native as nv, schedule as S
    Cin = 320
    g = torch.Generator().manual_seed(B * 7 + H)
    x = ((torch.randn(2 * B, H, W, Cin, generator=g).abs() * 0.7 - 0.2)).half().to(dev)
    w = (torch.randn(4, 9, Cin, generator=g) * (9 * Cin) ** -0.5).half().to(dev)
    b = (torch.randn(4, generator=g) * 0.2).half().to(dev)
    v_none, vc_none, _ = nv.op_conv_out_step(x, w, b)
    lams = torch.linspace(0.3, 7.5, B, dtype=torch.float32, device=dev)
    n_checked = 0
    for k, (method, dt, coef, uses_aux, slots) in enumerate(coef_variants()):
        kd = method == S.STEP_DPMPP2M_CFGPP
        scale = float(torch.tensor(1.0) / (torch.tensor(-coef.c0) ** 2 + 1) ** 0.5) if kd else None
        sdev = torch.tensor([scale], dtype=torch.float32, device=dev) if kd else None
        a, bb = (scale, float(torch.tensor(-coef.c0 * scale, dtype=torch.float32))) if kd else (coef.c1, coef.c0)
        z0 = (torch.randn(B, 4, H, W, generator=g) * 3).to(dt).to(dev)
        aux0 = torch.randn(B, 4, H, W, generator=g).to(dt).to(dev) if uses_aux else None
        noise = torch.randn(max(slots, 1), B, 4, H, W, generator=g).half().to(dev) if slots else None
        for lam in (None, lams):
            z, aux = z0.clone(), (aux0.clone() if uses_aux else None)
            v_uc, v_c, zt = nv.op_conv_out_step(x, w, b, method, coef, z, aux=aux, noise=noise, lambdas=lam,
                                                v_ab=(a, bb), in_scale=sdev)
            assert torch.equal(v_uc, v_none) and torch.equal(v_c, vc_none), "the v launch must write the raw output"
            e_uc, e_c = nv.op_v_to_eps(v_uc, z0, a, bb, sdev), nv.op_v_to_eps(v_c, z0, a, bb, sdev)
            assert torch.equal(e_uc, _v_to_eps_ref(v_uc, z0, a, bb, scale))
            zs, auxs = z0.clone(), (aux0.clone() if uses_aux else None)
            zts = nv.op_cfgpp_step(e_uc, e_c, method, coef, zs, aux=auxs, noise=noise, lambdas=lam)
            tag = f"v step {B}x{H}x{W} variant {k} (method {method}, {dt}, bits {coef.second_order}, " \
                  f"{'table' if lam is not None else 'scalar'})"
            assert torch.equal(z, zs) and torch.equal(zt, zts), tag
            if uses_aux:
                assert torch.equal(aux, auxs), tag + " aux"
            n_checked += 1
    print(f"[sd2] conv_out_step v {B}x{H}x{W}: {n_checked} variants bitwise equal to v_to_eps + standalone step")


# ---- the epsilon path is untouched -------------------------------------------------------------------------------

def test_prediction_type_zero_equals_legacy_handle():
    """cfgpp_create_ex with prediction_type = 0 and cfgpp_create (the layout without the field) run the same plan and
    kernels: predict_noise and the fused DDIM / DPM++ trajectories are bit-identical."""
    from ctypes import byref, c_int
    from cfgpp_b200 import _native as nv, config as C, kdiffusion as K, schedule as S, weights as Wt
    from cfgpp_b200.engine import NativeUNet

    class LegacyUNet(NativeUNet):
        def _create(self, desc, idx):
            nv.check(self.lib.cfgpp_create(byref(C.ModelDescC.from_buffer_copy(bytes(desc)[:C.ctypes.sizeof(
                C.ModelDescC)])), c_int(idx), byref(self._h)))

    cfg = C.tiny_sd2_config(prediction_type="epsilon")
    sd = Wt.synthetic_state_dict(cfg, seed=4, device=dev)
    g = torch.Generator().manual_seed(9)
    B, hw = 2, 32
    z = torch.randn(B, 4, hw, hw, generator=g).to(dev)
    ctx = torch.randn(2 * B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    sch = S.Schedule.make(5)
    sigmas = K.get_sigmas_karras(5, 0.0292, 14.6146, rho=7.)
    kd = S.kd_steps(sigmas, lambda s: torch.tensor(500), 0.6, True, second_order=True, diff_guided=True)
    outs = []
    for cls in (NativeUNet, LegacyUNet):
        net = cls(cfg, sd, dev)
        net.prepare(B, hw, hw)
        net.set_prompt(ctx)
        o = list(net.predict_noise(z, 601.0))
        net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, S.ddim_cfgpp_steps(sch, 0.6, False), [0.4, 0.9])
        net.set_state(z)
        net.run_steps()
        o += [net.get_state(0), net.get_state(1)]
        net.set_schedule(S.STEP_DPMPP2M_CFGPP, torch.float16, kd)
        net.set_state((z * 14.6).half())
        net.run_steps()
        o += [net.get_state(0), net.get_state(1), net.get_state(2)]
        outs.append(o)
        net.close()
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    print(f"[sd2] prediction_type 0 vs legacy cfgpp_create: {len(outs[0])} outputs bit-identical")


# ---- the SD 2 UNet -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,h,w,t", [(2, 96, 96, 801), (1, 64, 64, 401), (1, 96, 64, 21)])
def test_sd2_unet_full_geometry(B, h, w, t):
    """The real SD 2 UNet (865.9 M params, linear projections, 5 x 64 heads at the top level, context 1024) at 768^2
    (every level through the im2col conv A tile; 9216-token self-attention), 512^2 and 768 x 512."""
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    from oracle import unet as O
    cfg = C.sd2_config()
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    g = torch.Generator().manual_seed(B + h + w)
    z = torch.randn(B, 4, h, w, generator=g).to(dev)
    uc = torch.randn(B, 77, 1024, generator=g).half().to(dev)
    c = torch.randn(B, 77, 1024, generator=g).half().to(dev)
    net = NativeUNet(cfg, sd, dev)
    net.prepare(B, h, w)
    net.set_prompt(torch.cat([uc, c]))
    vu, vc = net.predict_noise(z, float(t))
    got = torch.cat([vu, vc]).float()
    net.close()
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
    ref16 = OracleCudaUNet(cfg, sd, dev)
    r16 = ref16(z_in, t_in, ctx)["sample"].float()
    del ref16
    m32 = O.build_unet(oracle_cfg(cfg), sd, dtype=torch.float32, device=dev)
    with torch.no_grad():
        r32 = m32(z_in, t_in, ctx.float())["sample"]
    del m32
    e16, e32, o32 = rel_l2(got, r16), rel_l2(got, r32), rel_l2(r16, r32)
    print(f"[sd2] UNet B={B} latent {h}x{w} t={t}: rel-L2 vs fp16 oracle {e16:.3e}, vs fp32 {e32:.3e} "
          f"(fp16 oracle vs fp32 {o32:.3e})")
    assert torch.isfinite(got).all() and e16 <= 5e-3 and e32 <= 1.5 * o32 + 1e-4


# ---- trajectories ---------------------------------------------------------------------------------------------------

def test_ddim_cfgpp_v_prediction_vs_oracle():
    """ddim_cfg++ on a v-prediction UNet: teacher-forced per step (the converted eps and z_{t-1}) <= 5e-3, free-running
    final Tweedie estimate <= 3e-2, against the oracle loop on the fp16-autocast oracle behind the stated v rule."""
    from cfgpp_b200 import config as C, schedule as S, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    from oracle import samplers as OSm, schedule as OS, sd2 as OV
    cfg = C.tiny_sd2_config()
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    net, ref = NativeUNet(cfg, sd, dev), OracleCudaUNet(cfg, sd, dev)
    B, hw, nfe, lam = 2, 32, 10, 0.6
    g = torch.Generator().manual_seed(7)
    z = torch.randn(B, 4, hw, hw, generator=g).to(dev)
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    tb = OS.make_tables(nfe)
    rec = []
    z0_ref = OSm.sd15_ddim_cfgpp(OV.VPredUNet(ref, OV.ddim_v_levels(tb)), tb, z, uc, c, lam, record=rec)
    steps = S.ddim_cfgpp_steps(S.Schedule.make(nfe), lam, sdxl_indexing=False)
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]))
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
    worst = 0.0
    for i, r in enumerate(rec):
        net.set_state(r["zt"])
        vu, vc = net.predict_noise(r["zt"], steps[i].t)
        a, b = net.v_coefs[i]
        eu, ec = S.v_to_eps(vu, r["zt"].half(), a, b), S.v_to_eps(vc, r["zt"].half(), a, b)
        errs = [rel_l2(eu, r["noise_uc"]), rel_l2(ec, r["noise_c"])]
        net.run_steps(i, 1)
        if i + 1 < len(rec):
            errs.append(rel_l2(net.get_state(0), rec[i + 1]["zt"]))
        worst = max(worst, *errs)
        assert max(errs) <= 5e-3, f"step {i}: {errs}"
    net.set_state(z)
    net.run_steps(0, nfe)
    e = rel_l2(net.get_state(1), z0_ref)
    print(f"[sd2] ddim_cfg++ v-pred NFE={nfe}: teacher-forced worst {worst:.3e}, free-running final z0t {e:.3e}")
    assert e <= 3e-2
    net.close()


@pytest.mark.parametrize("method", ["ddim_cfg++", "dpm++_2m_cfg++", "euler_a_cfg++"])
def test_fused_equals_callback_path_v_prediction(method):
    """With a callback installed the solvers run the un-fused seams (the DDIM callback loop, the op-by-op VE loops over
    _k_denoise), which convert v in torch with the same (a, b); the trajectories are bit-identical to the fused ones."""
    from cfgpp_b200 import config as C, latent_diffusion as LD
    cfg = C.tiny_sd2_config()
    solver = LD.get_solver(method, solver_config=SimpleNamespace(num_sampling=6), device=dev, unet_config=cfg,
                           model_key="synthetic:3", text_encoder=lambda p, d=None: None, vae=SimpleNamespace())
    g = torch.Generator().manual_seed(2)
    B = 2
    zT = torch.randn(B, 4, 32, 32, generator=g).to(dev)
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    lam = [0.4, 0.8]
    n_cb = []
    cb = lambda i, t, kw: n_cb.append(i) or kw  # noqa: E731
    outs = []
    for callback in (None, cb):
        torch.manual_seed(77)
        if method == "ddim_cfg++":
            outs.append([solver.reverse_process(uc, c, lam, zT.clone(), callback)])
        else:
            outs.append(list(solver.reverse_process(uc, c, lam, None, callback, noise=zT.clone())))
    assert n_cb, "the callback path did not run"
    assert all(torch.equal(a, b) for a, b in zip(*outs)), method
    print(f"[sd2] {method} v-pred: fused == callback path bit for bit ({len(n_cb)} callback steps)")


# ---- text tower -------------------------------------------------------------------------------------------------

def test_clip_h_against_transformers_on_gpu():
    """SD 2's OpenCLIP ViT-H as transformers' CLIPTextModel (fp16, as the reference loads it): last_hidden_state, what
    SD 2 conditions on, and the pooled output, on the same weights and ids."""
    tr = pytest.importorskip("transformers")
    from cfgpp_b200 import text_encoder as TE
    cfg = TE.clip_h_config()
    sd = TE.synthetic_clip_state_dict(cfg, seed=5, device=dev)
    hc = tr.CLIPTextConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                           num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                           max_position_embeddings=77, hidden_act=cfg.hidden_act, eos_token_id=2, bos_token_id=49406,
                           pad_token_id=1)
    ref = tr.CLIPTextModel(hc).eval()
    ref.load_state_dict({k: v.float().cpu() for k, v in sd.items()}, strict=False)
    g = torch.Generator().manual_seed(3)
    ids = torch.zeros(2, 77, dtype=torch.int32)  # "!" (id 0) pads after <|endoftext|>, as SD 2's tokenizer does
    for r, n in enumerate((9, 40)):
        ids[r, 0] = 49406
        ids[r, 1:n] = torch.randint(1, 49406, (n - 1,), generator=g, dtype=torch.int32)
        ids[r, n] = 49407
    with torch.no_grad():
        o = ref.to(device=dev, dtype=torch.float16)(ids.long().to(dev), output_hidden_states=True)
    enc = TE.NativeCLIPTextEncoder(cfg, sd, dev)
    hidden, last, pooled = enc.encode(ids, skip=1)
    for what, got, r in (("hidden_states[-2]", hidden, o.hidden_states[-2]), ("last_hidden_state", last, o.last_hidden_state),
                         ("pooler_output", pooled, o.pooler_output)):
        e = rel_l2(got, r)
        print(f"[sd2] clip_h vs transformers fp16 {what}: {e:.3e}")
        assert e <= 5e-3
    enc.close()


# ---- end to end -------------------------------------------------------------------------------------------------------

def test_sample_768_batched_per_image_guidance():
    """The SD 2.1 solver at its native 768^2 (synthetic weights): B = 4 prompts, one guidance scale per image."""
    from cfgpp_b200 import config as C, latent_diffusion as LD
    solver = LD.get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=4), device=dev,
                           unet_config=C.sd2_config(), model_key="synthetic:21")
    torch.manual_seed(0)
    img = solver.sample(cfg_guidance=[0.2, 0.4, 0.6, 0.8], prompt=["", ["a", "b", "c", "d"]])
    print(f"[sd2] sample() 768^2 B=4: shape {tuple(img.shape)}, mean {img.mean():.3f}")
    assert img.shape == (4, 3, 768, 768) and torch.isfinite(img).all()
    assert not torch.equal(img[0], img[3])


def test_inversion_example_sd20(tmp_path):
    """`python -m examples.inversion --model sd20`: encode -> CFG++ inversion -> reconstruction at 768^2."""
    out = subprocess.run([sys.executable, "-m", "examples.inversion", "--model", "sd20", "--NFE", "3",
                          "--cfg_guidance", "0.6", "--prompt", "a cat", "--workdir", str(tmp_path)],
                         cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    rec = torch.load(tmp_path / "result" / "reconstruct.pt")
    print(f"[sd2] examples.inversion --model sd20: {tuple(rec.shape)}, finite {bool(torch.isfinite(rec).all())}")
    assert rec.shape == (1, 3, 768, 768) and torch.isfinite(rec).all()
