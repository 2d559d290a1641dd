"""End-to-end images/s of `sample()` at batch 1, 2, 4 and 8 — the throughput a many-prompt run
(examples/text_to_mscoco.py --batch_size B) gets from putting B prompts into one trajectory.

    python tools/batch_throughput.py [--models sd15,sdxl] [--batches 1,2,4,8] [--nfe 50] [--reps 2] [--out FILE]
                                     [--height H --width W]

Each timed call is one `solver.sample()` with B distinct prompts: text encode, the fused trajectory (UNet batch 2B)
and the VAE decode, all on the native backend with seeded synthetic weights, then the images' copy to the host; the
clock stops after a device synchronise. Every batch size is warmed up with one untimed call first. SD v1.5 runs at
512² and SDXL at 1024² unless --height / --width pick another size (an SDXL aspect-ratio bucket, a non-square SD v1.5
size: the start latents are then drawn at that size and SDXL's size conditioning says so), all `ddim_cfg++` with
lambda = 0.6. The GPU's name, power limit and max SM clock are read in
the same process. Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def gpu_info() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        info["power_limit, max_sm_clock"] = q.stdout.strip() or q.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit, max_sm_clock"] = f"not read: {e}"
    return info


def make_solver(model: str, nfe: int):
    conf = SimpleNamespace(num_sampling=nfe)
    if model == "sd15":
        from cfgpp_b200.latent_diffusion import get_solver
        return get_solver("ddim_cfg++", solver_config=conf, device="cuda:0", model_key="synthetic:1234")
    from cfgpp_b200.latent_sdxl import get_solver
    return get_solver("ddim_cfg++", solver_config=conf, device="cuda:0", model_key="synthetic:1234")


def run_once(solver, model: str, batch: int, call: int, hw: tuple[int, int] | None = None):
    """One timed sample(); `hw` = (height, width) in pixels, or None for the model's native square size."""
    prompts = [f"a photograph of object {call * 8 + i}, studio light" for i in range(batch)]
    torch.manual_seed(1000 + call)
    kw = {}
    if hw is not None:
        h, w = hw
        kw["zT"] = torch.randn(batch, 4, h // 8, w // 8)
        if model != "sd15":
            kw.update(original_size=(h, w), target_size=(h, w))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if model == "sd15":
        img = solver.sample(cfg_guidance=0.6, prompt=["", prompts], **kw)
    else:
        img = solver.sample(prompt1=["", prompts], prompt2=["", prompts], cfg_guidance=0.6, **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert img.shape[0] == batch and torch.isfinite(img).all()
    if hw is not None:
        assert tuple(img.shape[-2:]) == hw
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="sd15,sdxl")
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--nfe", type=int, default=50)
    ap.add_argument("--reps", type=int, default=2, help="timed calls per batch size (after one warm-up call)")
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result here")
    ap.add_argument("--height", type=int, default=None,
                    help="image height in pixels (with --width; default: 512² for SD v1.5, 1024² for SDXL)")
    ap.add_argument("--width", type=int, default=None, help="image width in pixels (with --height)")
    args = ap.parse_args()
    if (args.height is None) != (args.width is None):
        ap.error("--height and --width go together")
    hw = (args.height, args.width) if args.height is not None else None
    if not torch.cuda.is_available():
        raise SystemExit("batch_throughput.py measures on a CUDA device; none is visible")
    batches = [int(b) for b in args.batches.split(",")]
    result = {"gpu": gpu_info(), "nfe": args.nfe, "method": "ddim_cfg++", "lambda": 0.6, "reps": args.reps,
              "timing": "host clock around sample() (text encode + trajectory + VAE decode + copy to host), "
                        "device synchronise before the clock stops, after one warm-up call per batch size",
              "models": {}}
    for model in args.models.split(","):
        solver = make_solver(model, args.nfe)
        rows = {}
        for b in batches:
            run_once(solver, model, b, call=0, hw=hw)  # warm-up: plan, graph capture, VAE / text plans for this shape
            times = [run_once(solver, model, b, call=1 + r, hw=hw) for r in range(args.reps)]
            best, worst = min(times), max(times)
            rows[b] = {"seconds_per_call": times, "images_per_s_best": b / best, "images_per_s_worst": b / worst}
            print(f"{model} B={b}: {b / best:.3f} img/s (best of {len(times)}; worst {b / worst:.3f})", flush=True)
        base = rows[batches[0]]["images_per_s_best"]
        for b in batches:
            rows[b]["speedup_vs_first"] = rows[b]["images_per_s_best"] / base
        native = 512 if model == "sd15" else 1024
        result["models"][model] = {"resolution": list(hw) if hw else native, "batches": rows}
        from cfgpp_b200 import latent_sdxl as LX
        del solver
        LX.release_engines()
        torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    line = json.dumps(result)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
