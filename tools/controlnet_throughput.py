"""The fused step with and without a ControlNet, at SD v1.5 512^2 batch 1 and 4 and SDXL 1024^2 batch 1:

    python tools/controlnet_throughput.py [--nfe 20] [--reps 3] [--out FILE]

Per configuration one engine on seeded synthetic weights runs a `ddim_cfg++` trajectory of NFE fused steps, first
uncontrolled, then with a ControlNet (synthetic, shaped like the base UNet) attached; the two alternate over `reps`
timed trajectories (CUDA events on the current stream around the NFE graph replays alone, the state set before the
window; after one warm-up trajectory of each). Reported per side: the
time of one fused step, the step FLOPs and launches per step from the plan's statistics, and the achieved FLOP/s; and
the controlled step's achieved FLOP/s over the uncontrolled one's. The once-per-image conditioning embedding is not a
step cost and is not timed. The GPU's name, power limit and max SM clock are read in the same process, before and
after. Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.batch_throughput import gpu_info  # noqa: E402
from tools.refiner_throughput import timed  # noqa: E402

CONFIGS = (("sd15", 1, 64), ("sd15", 4, 64), ("sdxl", 1, 128))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nfe", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3, help="timed trajectories of each side, alternating")
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("controlnet_throughput.py measures on a CUDA device; none is visible")
    from cfgpp_b200 import config as C, controlnet as CN, schedule as S, weights as Wt
    from cfgpp_b200.engine import NativeUNet

    result = {"gpu": gpu_info(), "method": "ddim_cfg++", "nfe": args.nfe, "reps": args.reps,
              "timing": "CUDA events around NFE fused steps (run_steps), after one warm-up trajectory each; "
                        "uncontrolled and controlled alternate", "configs": []}
    steps_cache = {}
    for name, B, hw in CONFIGS:
        cfg = C.CONFIGS[name]()
        eng = NativeUNet(cfg, Wt.synthetic_state_dict(cfg, seed=1234, device="cuda"), "cuda:0")
        cn_cfg = CN.controlnet_config(cfg)
        cn = CN.NativeControlNet(cn_cfg, CN.synthetic_controlnet_state_dict(cn_cfg, seed=99, device="cuda"), "cuda:0")
        torch.cuda.empty_cache()
        g = torch.Generator().manual_seed(0)
        zT = torch.randn(B, 4, hw, hw, generator=g).cuda()  # on the device: the timed window holds no upload
        uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
        c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
        pooled = tids = None
        if cfg.addition_embed_type == "text_time":
            pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().cuda()
            tids = torch.tensor([[8. * hw, 8. * hw, 0, 0, 8. * hw, 8. * hw]] * (2 * B)).cuda()
        image = torch.rand(B, 3, 8 * hw, 8 * hw, generator=g).cuda()
        key = (args.nfe, name)
        if key not in steps_cache:
            steps_cache[key] = S.ddim_cfgpp_steps(S.Schedule.make(args.nfe), 0.6,
                                                  sdxl_indexing=cfg.addition_embed_type is not None)
        steps = steps_cache[key]

        def setup(controlled: bool):
            eng.attach_controlnet(cn if controlled else None)
            eng.prepare(B, hw, hw)
            eng.bind_prompt(uc, c, pooled, tids, force=True)
            if controlled:
                eng.set_control_image(image)
            eng.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
            stats = dict(eng.plan_stats, launches_per_step=eng.launches_per_step)

            def traj():
                eng.run_steps(0, len(steps))
            eng.set_state(zT)
            traj()  # warm-up: captures the step graph
            torch.cuda.synchronize()
            return stats, traj

        sides = {}
        times = {False: [], True: []}
        for _ in range(args.reps):
            for controlled in (False, True):  # re-planned on every switch: each side keeps its own timed window
                stats, traj = setup(controlled)
                sides[controlled] = stats
                eng.set_state(zT)  # outside the timed window, which holds the NFE graph replays only
                times[controlled].append(timed(traj) / len(steps))
        assert torch.isfinite(eng.get_state(0)).all()
        row = {"model": name, "batch": B, "resolution": [8 * hw, 8 * hw]}
        for controlled, label in ((False, "uncontrolled"), (True, "controlnet")):
            ms = min(times[controlled])
            st = sides[controlled]
            row[label] = {"ms_per_step": times[controlled], "ms_per_step_best": ms, "step_flops": st["step_flops"],
                          "launches_per_step": st["launches_per_step"],
                          "tflops_per_s": st["step_flops"] / ms * 1e-9}
        row["achieved_flops_ratio"] = row["controlnet"]["tflops_per_s"] / row["uncontrolled"]["tflops_per_s"]
        print(f"{name} B={B} {8 * hw}^2: uncontrolled {row['uncontrolled']['ms_per_step_best']:.2f} ms/step "
              f"({row['uncontrolled']['tflops_per_s']:.0f} TFLOP/s, {row['uncontrolled']['launches_per_step']} "
              f"launches), ControlNet {row['controlnet']['ms_per_step_best']:.2f} ms/step "
              f"({row['controlnet']['tflops_per_s']:.0f} TFLOP/s, {row['controlnet']['launches_per_step']} launches); "
              f"achieved FLOP/s ratio {row['achieved_flops_ratio']:.3f}", flush=True)
        result["configs"].append(row)
        eng.close()
        cn.close()
        del eng, cn
        torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    line = json.dumps(result)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
