"""Shared helpers of the GPU parity tests: oracle construction, seeded inputs, error metrics."""
import dataclasses

import torch

from cfgpp_b200 import config as C
from cfgpp_b200 import weights as Wt
from oracle import unet as O


def oracle_cfg(cfg):
    return O.UNetConfig(**{f.name: getattr(cfg, f.name) for f in dataclasses.fields(O.UNetConfig)})


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def make_inputs(cfg, B, hw, device, seed=7, duplicate_added=True):
    g = torch.Generator(device="cpu").manual_seed(seed)
    z = torch.randn(B, 4, hw, hw, generator=g).to(device)
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(device)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(device)
    add = None
    if cfg.addition_embed_type == "text_time":
        rows = 2 * B if duplicate_added else B
        pooled = torch.randn(rows, cfg.pooled_dim, generator=g).half().to(device)
        tid = torch.tensor([[hw * 8, hw * 8, 0, 0, hw * 8, hw * 8]] * rows, dtype=torch.float16).to(device)
        add = {"text_embeds": pooled, "time_ids": tid}
    return z, uc, c, add


class OracleCudaUNet:
    """The restated UNet under torch.autocast('cuda', fp16) with fp16 weights == stand-in for the reference's CUDA
    path (same torch op sequence)."""
    def __init__(self, cfg, sd, device):
        self.m = O.build_unet(oracle_cfg(cfg), sd, dtype=torch.float16, device=device)

    def __call__(self, z, t, encoder_hidden_states=None, added_cond_kwargs=None):
        with torch.autocast("cuda", dtype=torch.float16), torch.no_grad():
            return self.m(z, t, encoder_hidden_states, added_cond_kwargs)


def coef_variants():
    """(method, state dtype, coef, uses aux, noise slots) over every step mode and second_order bit."""
    from cfgpp_b200 import kdiffusion as K, schedule as S
    sch = S.Schedule.make(20)
    out = []
    for dt in (torch.float32, torch.float16):
        out.append((S.STEP_DDIM_CFGPP, dt, S.ddim_cfgpp_steps(sch, 0.6, True)[7].coef, False, 0))
        out.append((S.STEP_DDIM_INV_CFGPP, dt, S.ddim_inversion_cfgpp_steps(sch, 0.6)[5].coef, False, 0))
        out.append((S.STEP_DDIM_CFG, dt, S.ddim_cfgpp_steps(sch, 0.6, True)[11].coef, False, 0))
        sigmas = K.get_sigmas_karras(6, 0.03, 14.6, rho=7.)
        ts = lambda s: torch.tensor(500)  # noqa: E731
        for cfgpp in (True, False):
            for second, diff in ((False, False), (True, False), (True, True)):
                for st in S.kd_steps(sigmas, ts, 0.6, cfgpp, second_order=second, diff_guided=diff)[:3]:
                    out.append((S.STEP_DPMPP2M_CFGPP, dt, st.coef, True, 0))
            for two_s in (False, True):
                steps, slots = S.kd_ancestral_steps(sigmas, ts, 0.6, cfgpp, two_s)
                for st in steps[:3]:
                    out.append((S.STEP_DPMPP2M_CFGPP, dt, st.coef, True, slots))
    bits = {v[2].second_order for v in out if v[0] == S.STEP_DPMPP2M_CFGPP}
    assert {b_ for b in bits for b_ in (1, 2, 4, 8, 16, 32) if b & b_} == {1, 2, 4, 8, 16, 32}
    return out


def build_pair(name, device, seed=1234):
    """(cfg, state_dict, native engine, fp16-autocast oracle) for a named config."""
    from cfgpp_b200.engine import NativeUNet
    cfg = C.CONFIGS[name]()
    sd = Wt.synthetic_state_dict(cfg, seed=seed, device=device)
    return cfg, sd, NativeUNet(cfg, sd, device), OracleCudaUNet(cfg, sd, device)
