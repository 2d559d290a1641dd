"""Stable Diffusion 2.1 at 768^2: images/s of `ddim_cfg++` (NFE 50) at batch 1 and 4, and how much of the UNet's
3x3-convolution time goes through the im2col A tile (at latent 96 the level widths 96 / 48 / 24 / 12 fit no tiled TMA
box).

    python tools/sd2_throughput.py [--batches 1,4] [--nfe 50] [--reps 2] [--out FILE]

Each timed call is one `solver.sample()` with B distinct prompts (ViT-H text encode, the fused v-prediction
trajectory at UNet batch 2B, the VAE decode, the copy to the host), seeded synthetic weights, after one untimed
warm-up call per batch size; the clock stops after a device synchronise. The convolution split comes from one
profiled eager forward (CUDA events around every plan entry) at batch 1: an entry is an im2col convolution when the
schedule its geometry gets (`cfgpp_dbg_gemm_schedule`) takes the im2col A tile. The GPU's name, power limit and max SM
clock are read in the same process. Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import re
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.batch_throughput import gpu_info  # noqa: E402


def conv_modes(cfg, h: int, w: int, batch: int) -> dict:
    """{(level, stride): a_mode} of the UNet's 3x3 convolutions at latent h x w (UNet batch 2 * batch)."""
    from cfgpp_b200 import _native as nv
    out = {}
    for lvl, ch in enumerate(cfg.block_out_channels):
        H, W = h >> lvl, w >> lvl
        x = torch.zeros(2 * batch, H, W, ch, dtype=torch.float16, device="cuda:0")
        wp = torch.zeros(ch, 9 * ch, dtype=torch.float16, device="cuda:0")
        for stride in (1, 2):
            out[(lvl, stride)] = nv.conv3x3_schedule(x, wp, stride=stride)["a_mode"]
    return out


def entry_level(name: str, levels: int):
    """(level, stride) of a conv plan entry by its diffusers module path, or None."""
    m = re.match(r"down_blocks\.(\d+)\.", name)
    if m:
        return int(m.group(1)), 2 if "downsamplers" in name else 1
    m = re.match(r"up_blocks\.(\d+)\.", name)
    if m:
        lvl = levels - 1 - int(m.group(1))
        return (lvl - 1, 1) if "upsamplers" in name else (lvl, 1)
    if name.startswith("mid_block"):
        return levels - 1, 1
    return None


def conv_split(solver, h: int, w: int) -> dict:
    eng = solver.unet
    eng.prepare(1, h, w)
    ctx = torch.randn(2, 77, solver.cfg.cross_attention_dim, device="cuda:0").half()
    eng.set_prompt(ctx)
    z = torch.randn(1, 4, h, w, device="cuda:0")
    eng.profile_forward(z, 501.0)  # warm-up
    prof = eng.profile_forward(z, 501.0)
    modes = conv_modes(solver.cfg, h, w, 1)
    total = sum(ms for _, _, _, ms in prof)
    conv = {"im2col": 0.0, "tiled": 0.0, "unclassified": 0.0}
    for name, kind, _, ms in prof:
        if kind != 1:
            continue
        key = entry_level(name, len(solver.cfg.block_out_channels))
        conv[modes[key] if key in modes else "unclassified"] += ms
    conv_ms = sum(conv.values())
    return {"forward_ms_eager_profiled": total, "conv3x3_ms": conv_ms, "conv3x3_share_of_forward": conv_ms / total,
            "im2col_share_of_conv3x3": conv["im2col"] / conv_ms if conv_ms else 0.0, "conv3x3_ms_by_a_mode": conv,
            "a_mode_by_level_stride": {f"{k[0]}/s{k[1]}": v for k, v in modes.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--nfe", type=int, default=50)
    ap.add_argument("--reps", type=int, default=2, help="timed calls per batch size (after one warm-up call)")
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sd2_throughput.py measures on a CUDA device; none is visible")
    from cfgpp_b200 import config as C
    from cfgpp_b200.latent_diffusion import get_solver
    solver = get_solver("ddim_cfg++", solver_config=SimpleNamespace(num_sampling=args.nfe), device="cuda:0",
                        unet_config=C.sd2_config(), model_key="synthetic:1234")
    result = {"gpu": gpu_info(), "model": "sd2.1 (v-prediction), synthetic weights", "resolution": [768, 768],
              "nfe": args.nfe, "method": "ddim_cfg++", "lambda": 0.6, "reps": args.reps,
              "timing": "host clock around sample() (text encode + trajectory + VAE decode + copy to host), device "
                        "synchronise before the clock stops, after one warm-up call per batch size", "batches": {}}
    for b in [int(x) for x in args.batches.split(",")]:
        times = []
        for call in range(args.reps + 1):
            prompts = [f"a photograph of object {call * 8 + i}, studio light" for i in range(b)]
            torch.manual_seed(1000 + call)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            img = solver.sample(cfg_guidance=0.6, prompt=["", prompts])
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert img.shape == (b, 3, 768, 768) and torch.isfinite(img).all()
            if call:
                times.append(dt)
        result["batches"][b] = {"seconds_per_call": times, "images_per_s_best": b / min(times),
                                "images_per_s_worst": b / max(times)}
        print(f"sd2.1 768^2 B={b}: {b / min(times):.3f} img/s (best of {len(times)})", flush=True)
    result["conv"] = conv_split(solver, 96, 96)
    result["gpu_after"] = gpu_info()
    line = json.dumps(result)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
