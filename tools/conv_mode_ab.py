"""CUDA-event time of the implicit-GEMM 3x3 convolutions with the tiled A tile and with the im2col A tile forced, at the
conv shapes of the SDXL UNet at 1024² (latent 128 x 128, UNet batch 2) — the A/B behind the choice of mode in
`make_conv3x3_op` (tiled wherever it can address the geometry).

    python tools/conv_mode_ab.py [--iters 50] [--rounds 5] [--out FILE]

Each shape runs both modes alternately for `rounds` rounds of `iters` back-to-back launches between two CUDA events
(after a warm-up of both); the table gives the median microseconds per launch and the spread over rounds, the
outputs of the two modes are checked to be bit-identical. The GPU's name and power limit are read in the same process.
Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.batch_throughput import gpu_info  # noqa: E402

# (B, H, W, Cin, Cout, stride): the SDXL UNet's conv3x3 shapes at latent 128 x 128, UNet batch 2
SHAPES = [
    (2, 128, 128, 320, 320, 1),    # down 0 / up 2 resnets
    (2, 128, 128, 640, 320, 1),    # up 2 resnet conv1 on cat(h, skip)
    (2, 128, 128, 320, 320, 2),    # down 0 Downsample2D
    (2, 64, 64, 320, 640, 1),      # down 1 resnet 0 conv1
    (2, 64, 64, 640, 640, 1),
    (2, 64, 64, 1280, 640, 1),     # up 1 resnet conv1 on cat(h, skip)
    (2, 64, 64, 640, 640, 2),      # down 1 Downsample2D
    (2, 32, 32, 640, 1280, 1),
    (2, 32, 32, 1280, 1280, 1),
    (2, 32, 32, 2560, 1280, 1),    # up 0 resnet conv1 on cat(h, skip)
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv_mode_ab.py measures on a CUDA device; none is visible")
    from cfgpp_b200 import _native as nv
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for B, H, W, Cin, Cout, s in SHAPES:
        x = torch.randn(B, H, W, Cin, generator=g, device=dev).half()
        w = (torch.randn(Cout, 9 * Cin, generator=g, device=dev) * (9 * Cin) ** -0.5).half()
        bias = torch.randn(Cout, generator=g, device=dev).half()
        run = {m: (lambda m=m: nv.op_conv3x3_ex(x, w, bias, stride=s, force_im2col=(m == "im2col")))
               for m in ("tiled", "im2col")}
        outs = {m: f() for m, f in run.items()}
        assert torch.equal(outs["tiled"], outs["im2col"]), f"modes differ at {B}x{H}x{W} {Cin}->{Cout} s{s}"
        us = {m: [] for m in run}
        for _ in range(args.rounds):
            for m, f in run.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    f()
                e1.record()
                e1.synchronize()
                us[m].append(e0.elapsed_time(e1) * 1e3 / args.iters)
        flops = 2.0 * B * (H // s) * (W // s) * Cout * 9 * Cin
        row = {"shape": f"{B}x{H}x{W} {Cin}->{Cout} stride {s}"}
        for m in run:
            med = statistics.median(us[m])
            row[m] = {"us_median": med, "us_min": min(us[m]), "us_max": max(us[m]), "tflops": flops / med * 1e-6}
        row["im2col_over_tiled"] = row["im2col"]["us_median"] / row["tiled"]["us_median"]
        rows.append(row)
        print(f"{row['shape']:32s} tiled {row['tiled']['us_median']:8.1f} us "
              f"[{row['tiled']['us_min']:.1f}, {row['tiled']['us_max']:.1f}]   im2col {row['im2col']['us_median']:8.1f} us "
              f"[{row['im2col']['us_min']:.1f}, {row['im2col']['us_max']:.1f}]   ratio {row['im2col_over_tiled']:.3f}",
              flush=True)
    line = json.dumps({"gpu": gpu_info(), "iters": args.iters, "rounds": args.rounds, "rows": rows})
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
