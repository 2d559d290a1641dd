"""Every output of every registered solver, on seeded synthetic weights, in one file: the check that a change to the
solver layer (latent_diffusion.py, latent_sdxl.py, kdiffusion.py, engine.py) computes what the tree before it did.

    python tools/solver_outputs.py --root TREE --out FILE      # TREE: the directory holding the cfgpp_b200 to import
    python tools/solver_outputs.py --compare OLD.pt NEW.pt     # every tensor torch.equal, same keys, same errors

To compare against an earlier commit, export its package (`git archive <commit> cfgpp_b200 | tar -x -C old`) and run
both trees on one native library (`CFGPP_B200_LIB=cfgpp_b200/lib/libcfgpp_b200.so`), or each on its own build when
the change is to the library. Covered: both registries on the tiny SD v1.5 and SDXL configs, three SD solvers on the
tiny v-prediction SD 2 config, and the SDXL solvers that take a refiner with a tiny refiner. Per solver: `sample()` (B = 2 prompts, per-image guidance [0.6, 1.0] where the solver
takes it; Lightning at 1.0), `reverse_process()` fused, `reverse_process()` under an identity callback with every
(t, z0t, zt) it saw, and `inversion()`; every call after `torch.manual_seed(0)`. ControlNet: `sample()` with a
synthetic ControlNet whose scale differs between schedule entries, fused and under the identity callback, for a
deterministic and an ancestral SD v1.5 and SD 2 method and two SDXL methods (SDXL has no ancestral one). Needs a CUDA
device."""
from __future__ import annotations

import argparse
import sys
from types import SimpleNamespace

import torch

SD2_SOLVERS = ("ddim_cfg++", "ddim_inversion_cfg++", "dpm++_2s_a_cfg++")
HW, B, LAM = 32, 2, [0.6, 1.0]
# 5 steps from 0.2 to 0.8: the first and last entries run unconditioned, the others at 0.7
CONTROL = dict(controlnet_conditioning_scale=0.7, control_guidance_start=0.2, control_guidance_end=0.8)


class Recorder:
    """Identity callback that keeps what it was shown."""
    def __init__(self):
        self.seen = []

    def __call__(self, i, t, kw):
        self.seen += [torch.as_tensor(t), kw['z0t'].clone(), kw['zt'].clone()]
        return kw


def _flat(x):
    return [x] if torch.is_tensor(x) else [t for e in x for t in _flat(e)]


class Outputs(dict):
    def call(self, key, fn):
        torch.manual_seed(0)
        cb = Recorder()
        try:
            res = fn(cb)
        except Exception as e:  # an error is an output too: both trees must raise it
            self.setdefault("errors", {})[key] = f"{type(e).__name__}: {e}"
            return
        for j, t in enumerate(_flat(res) + cb.seen):
            self[f"{key}/{j}"] = t.detach().cpu()


def sd_outputs(out: Outputs, dev):
    from cfgpp_b200 import config as C, latent_diffusion as LD
    jobs = [(C.tiny_sd15_config(), n) for n in LD.__SOLVER__] + [(C.tiny_sd2_config(), n) for n in SD2_SOLVERS]
    for cfg, name in jobs:
        s = LD.get_solver(name, solver_config=SimpleNamespace(num_sampling=5), device=dev, unet_config=cfg,
                          model_key="synthetic:11")
        g = torch.Generator().manual_seed(1)
        uc, c = (torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev) for _ in range(2))
        z = torch.randn(B, 4, HW, HW, generator=g).to(dev)
        src = torch.rand(1, 3, 8 * HW, 8 * HW, generator=g) * 2 - 1
        key = f"{cfg.name}/{name}"
        if "inversion" in name or "edit" in name:
            out.call(f"{key}/sample", lambda cb: s.sample(src, cfg_guidance=0.6, prompt=["", "a cat", "a dog"]))
        else:
            out.call(f"{key}/sample", lambda cb: s.sample(cfg_guidance=LAM, prompt=["", ["a cat", "a dog"]]))
        out.call(f"{key}/reverse", lambda cb: s.reverse_process(uc, c, LAM, z.clone()))
        out.call(f"{key}/reverse_cb", lambda cb: s.reverse_process(uc, c, LAM, z.clone(), cb))
        out.call(f"{key}/inversion", lambda cb: s.inversion(z[:1].half(), uc[:1], c[:1], 0.6))


def sdxl_outputs(out: Outputs, dev):
    from cfgpp_b200 import config as C, latent_sdxl as LX
    cfg = C.tiny_sdxl_config()
    refiner = LX.SDXLRefiner(model_key="synthetic:13", device=dev, unet_config=C.tiny_sdxl_refiner_config())
    for name in LX.__SOLVER__:
        light = name.endswith("lightning")
        kw = dict(solver_config=SimpleNamespace(num_sampling=4 if light else 5), device=dev, unet_config=cfg)
        s = LX.get_solver(name, **kw) if light else LX.get_solver(name, model_key="synthetic:12", **kw)
        lam = 1.0 if light else LAM
        g = torch.Generator().manual_seed(2)
        uc, c, c2 = (torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev) for _ in range(3))
        pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().to(dev)
        tids = torch.tensor([[8. * HW] * 2 + [0.] * 2 + [8. * HW] * 2] * (2 * B), device=dev)
        add = lambda rows=2 * B: {'text_embeds': pooled[:rows], 'time_ids': tids[:rows]}  # noqa: E731
        z = torch.randn(B, 4, HW, HW, generator=g).to(dev)
        src = torch.rand(1, 3, 8 * HW, 8 * HW, generator=g) * 2 - 1
        p1, p2 = ["", ["a cat", "a dog"]], ["", ["a cat", "a dog"]]
        key = f"{cfg.name}/{name}"
        if "edit" in name:
            p3 = ["", "a cat", "a dog"]
            out.call(f"{key}/sample", lambda cb: s.sample(p3, p3, cfg_guidance=0.6, src_img=src))
            rev = lambda cb: s.reverse_process(uc[:1], c[:1], c2[:1], 0.6, add(2), add(2), cb, src_img=src)  # noqa: E731
            out.call(f"{key}/reverse", lambda cb: rev(None))
            out.call(f"{key}/reverse_cb", rev)
        else:
            out.call(f"{key}/sample", lambda cb: s.sample(p1, p2, cfg_guidance=lam))
            out.call(f"{key}/reverse", lambda cb: s.reverse_process(uc, c, lam, add(), (8 * HW, 8 * HW), zT=z.clone()))
            out.call(f"{key}/reverse_cb", lambda cb: s.reverse_process(uc, c, lam, add(), (8 * HW, 8 * HW), cb,
                                                                       zT=z.clone()))
        out.call(f"{key}/inversion", lambda cb: s.inversion(z[:1].half(), uc[:1], c[:1], 0.6, add(2)))
        if name in LX.REFINER_SOLVERS:  # at 5 steps (DPM++: 4) a hand-off at 0.5 leaves each expert two or more
            ref = lambda cb: s.sample(p1, p2, cfg_guidance=LAM, refiner=refiner, denoising_end=0.5,  # noqa: E731
                                      callback_fn=cb)
            out.call(f"{key}/refiner", lambda cb: ref(None))
            out.call(f"{key}/refiner_cb", ref)


def controlnet_outputs(out: Outputs, dev):
    from cfgpp_b200 import config as C, controlnet as CN, latent_diffusion as LD, latent_sdxl as LX
    jobs = [(LD, C.tiny_sd15_config(), ("ddim_cfg++", "euler_a_cfg++")),
            (LD, C.tiny_sd2_config(), ("ddim_cfg++", "dpm++_2s_a_cfg++")),
            (LX, C.tiny_sdxl_config(), ("ddim_cfg++", "dpm++_2m_cfgpp"))]
    for family, cfg, names in jobs:
        cn = CN.ControlNet("synthetic-controlnet", dev, base_cfg=cfg)  # controlnet.synthetic_controlnet_state_dict
        image = torch.rand(1, 3, 8 * HW, 8 * HW, generator=torch.Generator().manual_seed(3))
        ctl = dict(controlnet=cn, control_image=image, **CONTROL)
        p = ["", ["a cat", "a dog"]]
        for name in names:
            s = family.get_solver(name, solver_config=SimpleNamespace(num_sampling=5), device=dev, unet_config=cfg,
                                  model_key="synthetic:14")
            if family is LD:
                run = lambda cb: s.sample(cfg_guidance=LAM, prompt=p, callback_fn=cb, **ctl)  # noqa: E731
            else:
                run = lambda cb: s.sample(p, p, cfg_guidance=LAM, callback_fn=cb, **ctl)  # noqa: E731
            key = f"{cfg.name}/controlnet/{name}"
            out.call(f"{key}/sample", lambda cb: run(None))
            out.call(f"{key}/sample_cb", run)
        cn.engine.close()


def compare(a_path: str, b_path: str) -> int:
    a, b = torch.load(a_path), torch.load(b_path)
    bad = sorted(set(a) ^ set(b))
    if a.get("errors") != b.get("errors"):
        bad.append(f"errors differ: {a.get('errors')} vs {b.get('errors')}")
    keys = [k for k in sorted(set(a) & set(b)) if k != "errors"]
    bad += [k for k in keys if a[k].dtype != b[k].dtype or not torch.equal(a[k], b[k])]
    print(f"{len(keys)} tensors compared, {len(bad)} mismatches; errors raised by both: {len(a.get('errors', {}))}")
    for k in bad:
        print("  MISMATCH", k)
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--root", default=".")
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    sys.path.insert(0, args.root)
    import cfgpp_b200
    print(f"solver outputs of {cfgpp_b200.__file__}")
    out, dev = Outputs(), torch.device("cuda:0")
    with torch.no_grad():
        sd_outputs(out, dev)
        sdxl_outputs(out, dev)
        controlnet_outputs(out, dev)
    torch.save(dict(out), args.out)
    print(f"{len(out) - ('errors' in out)} tensors -> {args.out}; errors: {out.get('errors', {})}")


if __name__ == "__main__":
    main()
