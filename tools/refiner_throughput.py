"""SDXL base-only against the base + refiner ensemble at 1024^2, batch 2, `ddim_cfg++`, lambda 0.6, NFE 50:

    A: the base UNet for all 50 steps
    B: the base for steps [0, 40), the refiner for [40, 50) (denoising_end 0.8), one fused trajectory with the
       device-side hand-off

    python tools/refiner_throughput.py [--nfe 50] [--reps 5] [--out FILE]

Each timed call is one `reverse_process()` (the fused trajectory and nothing else: no text encode, no VAE decode)
on seeded synthetic weights and conditioning, timed with CUDA events on the current stream after one untimed warm-up
call of each; A and B alternate so that drift of the shared host or clock hits both alike. Per model it reports the
time of one fused step (a whole NFE-step trajectory on that engine alone over NFE), `forward_flops` per forward, the
plan's workspace, the fp16 parameter bytes and the device memory the engine took when it was created. The GPU's name,
power limit and max SM clock are read in the same process, before and after. Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import math
import sys
from pathlib import Path
from types import SimpleNamespace

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.batch_throughput import gpu_info  # noqa: E402


def timed(fn, reps: int = 1) -> float:
    """ms of `fn` on the current stream, by CUDA events."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def conditioning(cfg, B: int, g, last):
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
    pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().cuda()
    tids = torch.tensor([[1024., 1024., 0., 0., *l] for l in last], dtype=torch.float16).cuda()
    return uc, c, {"text_embeds": pooled, "time_ids": tids}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nfe", type=int, default=50)
    ap.add_argument("--denoising_end", type=float, default=0.8)
    ap.add_argument("--reps", type=int, default=5, help="timed calls of A and of B, alternating")
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("refiner_throughput.py measures on a CUDA device; none is visible")
    from cfgpp_b200 import config as C, schedule as S, weights as Wt
    from cfgpp_b200.conditioning import SyntheticTextEncoder
    from cfgpp_b200.latent_sdxl import SDXLRefiner, get_solver

    B, hw, lam = 2, 128, 0.6
    result = {"gpu": gpu_info(), "resolution": [1024, 1024], "batch": B, "method": "ddim_cfg++", "lambda": lam,
              "nfe": args.nfe, "denoising_end": args.denoising_end, "reps": args.reps,
              "timing": "CUDA events around reverse_process() (fused trajectory only), after one warm-up call each; "
                        "A and B alternate"}

    def free_bytes():  # the synthetic state dicts are freed once loaded: return PyTorch's cache before reading
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return torch.cuda.mem_get_info()[0]

    free0 = free_bytes()
    solver = get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=args.nfe), device="cuda:0",
                        model_key="synthetic:1234", vae=SimpleNamespace(),
                        text_encoders=(SyntheticTextEncoder(768, 0), SyntheticTextEncoder(1280, 1280)))
    free1 = free_bytes()
    refiner = SDXLRefiner(model_key="synthetic:4321", device="cuda:0")
    free2 = free_bytes()

    g = torch.Generator().manual_seed(0)
    zT = torch.randn(B, 4, hw, hw, generator=g)
    base_c = conditioning(solver.cfg, B, g, [(1024., 1024.)] * (2 * B))
    ref_c = conditioning(refiner.cfg, B, g, [(2.5,)] * B + [(6.0,)] * B)
    k = S.expert_split(solver._sch.timesteps, args.denoising_end, args.nfe)

    def run_a():
        return solver.reverse_process(base_c[0], base_c[1], lam, base_c[2], (1024, 1024), None, zT=zT)

    def run_b():
        return solver.reverse_process(base_c[0], base_c[1], lam, base_c[2], (1024, 1024), None, zT=zT,
                                      refiner=refiner, refiner_cond=ref_c, denoising_end=args.denoising_end)

    for fn in (run_a, run_b):  # warm-up: plans, graphs, prompt binding
        fn()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(args.reps):
        ta.append(timed(run_a))
        tb.append(timed(run_b))
    za, zb = run_a(), run_b()
    assert torch.isfinite(za).all() and torch.isfinite(zb).all()

    # one fused step per model: a whole trajectory on that engine alone (its plan and prompt stay bound)
    steps = S.ddim_cfgpp_steps(solver._sch, lam, sdxl_indexing=True)
    models = {}
    for name, eng, cfg, cond, free_before, free_after in (
            ("sdxl_base", solver.unet, solver.cfg, base_c, free0, free1),
            ("sdxl_refiner", refiner.unet, refiner.cfg, ref_c, free1, free2)):
        eng.prepare(B, hw, hw)
        eng.bind_prompt(cond[0], cond[1], cond[2]["text_embeds"], cond[2]["time_ids"], force=True)
        eng.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)

        def traj():
            eng.set_state(zT)
            eng.run_steps(0, len(steps))
        traj()
        ms = min(timed(traj) for _ in range(3)) / len(steps)
        f = eng.forward_flops
        models[name] = {"ms_per_fused_step": ms, "forward_flops": f, "tflops_per_s": f / ms * 1e-9,
                        "workspace_bytes": eng.workspace_bytes,
                        "param_bytes_fp16": 2 * sum(math.prod(s) for _, s, _ in Wt.unet_param_specs(cfg)),
                        "device_bytes_at_create": free_before - free_after}
        print(f"{name}: {ms:.2f} ms per fused step (UNet batch {2 * B}), {f / 1e12:.2f} TFLOP per forward, "
              f"workspace {eng.workspace_bytes / 2**30:.2f} GiB", flush=True)
    result["models"] = models
    ma, mb = min(ta), min(tb)
    result["A_base_only"] = {"ms": ta, "ms_best": ma, "images_per_s_best": B / ma * 1e3}
    result["B_base_plus_refiner"] = {"ms": tb, "ms_best": mb, "images_per_s_best": B / mb * 1e3,
                                     "base_steps": k, "refiner_steps": args.nfe - k}
    result["B_over_A"] = mb / ma
    result["gpu_after"] = gpu_info()
    print(f"A base-only NFE {args.nfe}: {ma:.1f} ms; B base {k} + refiner {args.nfe - k}: {mb:.1f} ms "
          f"(B / A = {mb / ma:.3f})", flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
