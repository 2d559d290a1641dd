"""The fused step with and without T2I-Adapter features, at SD v1.5 512^2 batch 4 and SDXL 1024^2 batch 1, and the
adapter's own forward:

    python tools/t2i_adapter_throughput.py [--nfe 20] [--reps 5] [--out FILE]

Per configuration one engine on seeded synthetic weights runs a `ddim_cfg++` trajectory of NFE fused steps, without
features, then with a synthetic adapter's features attached; the two alternate over `reps` timed trajectories (CUDA events
on the current stream around the NFE graph replays alone, after one warm-up trajectory of each; best of `reps`).
Reported per side: ms per fused step and launches per step; and the difference. The adapter forward (once per image,
not a step cost) is timed on its own at 1 and 8 images, best of `reps` after a warm-up, as ms per image. The GPU's
name, power limit and max SM clock are read in the same process, before and after. Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.batch_throughput import gpu_info  # noqa: E402
from tools.refiner_throughput import timed  # noqa: E402

CONFIGS = (("sd15", 4, 64), ("sdxl", 1, 128))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nfe", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5, help="timed trajectories of each side, alternating")
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("t2i_adapter_throughput.py measures on a CUDA device; none is visible")
    from cfgpp_b200 import config as C, schedule as S, t2i_adapter as T, weights as Wt
    from cfgpp_b200.engine import NativeUNet

    result = {"gpu": gpu_info(), "method": "ddim_cfg++", "nfe": args.nfe, "reps": args.reps,
              "timing": "CUDA events around NFE fused steps (run_steps), after one warm-up trajectory each; without "
                        "and with features alternate; best of reps", "configs": []}
    for name, B, hw in CONFIGS:
        cfg = C.CONFIGS[name]()
        eng = NativeUNet(cfg, Wt.synthetic_state_dict(cfg, seed=1234, device="cuda"), "cuda:0")
        acfg = T.t2i_adapter_config(cfg)
        ad = T.NativeT2IAdapter(acfg, T.synthetic_t2i_adapter_state_dict(acfg, seed=77, device="cuda"), "cuda:0")
        g = torch.Generator().manual_seed(0)
        zT = torch.randn(B, 4, hw, hw, generator=g).cuda()
        uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
        c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
        pooled = tids = None
        if cfg.addition_embed_type == "text_time":
            pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().cuda()
            tids = torch.tensor([[8. * hw, 8. * hw, 0, 0, 8. * hw, 8. * hw]] * (2 * B)).cuda()
        image = torch.rand(8, 3, 8 * hw, 8 * hw, generator=g).cuda()
        feats = ad.features(image[:B].contiguous())
        steps = S.ddim_cfgpp_steps(S.Schedule.make(args.nfe), 0.6, sdxl_indexing=cfg.addition_embed_type is not None)

        def setup(with_t2i: bool):
            eng.attach_t2i(len(feats) if with_t2i else 0)
            eng.prepare(B, hw, hw)
            eng.bind_prompt(uc, c, pooled, tids, force=True)
            if with_t2i:
                eng.set_t2i_features(feats)
            eng.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
            launches = eng.launches_per_step

            def traj():
                eng.run_steps(0, len(steps))
            eng.set_state(zT)
            traj()  # warm-up: captures the step graph
            torch.cuda.synchronize()
            return launches, traj

        launches, times = {}, {False: [], True: []}
        for _ in range(args.reps):
            for with_t2i in (False, True):
                launches[with_t2i], traj = setup(with_t2i)
                eng.set_state(zT)  # outside the timed window
                times[with_t2i].append(timed(traj) / len(steps))
        assert torch.isfinite(eng.get_state(0)).all()
        row = {"model": name, "batch": B, "resolution": [8 * hw, 8 * hw]}
        for with_t2i, label in ((False, "plain"), (True, "t2i_adapter")):
            row[label] = {"ms_per_step": times[with_t2i], "ms_per_step_best": min(times[with_t2i]),
                          "launches_per_step": launches[with_t2i]}
        row["added_ms_per_step"] = row["t2i_adapter"]["ms_per_step_best"] - row["plain"]["ms_per_step_best"]
        adapter = {}
        for nb in (1, 8):
            img = image[:nb].contiguous()
            ad.features(img)  # warm-up: builds the plan for this batch
            torch.cuda.synchronize()
            adapter[str(nb)] = min(timed(lambda: ad.features(img)) for _ in range(args.reps)) / nb
        row["adapter_ms_per_image"] = adapter
        row["adapter_gflops_per_image"] = ad.stats["flops"] / 8 * 1e-9
        print(f"{name} B={B} {8 * hw}^2: plain {row['plain']['ms_per_step_best']:.3f} ms/step "
              f"({row['plain']['launches_per_step']} launches), with features "
              f"{row['t2i_adapter']['ms_per_step_best']:.3f} ms/step ({row['t2i_adapter']['launches_per_step']} "
              f"launches), +{row['added_ms_per_step'] * 1e3:.1f} us; adapter {adapter['1']:.3f} ms/image at 1, "
              f"{adapter['8']:.3f} ms/image at 8", flush=True)
        result["configs"].append(row)
        eng.close()
        ad.close()
        del eng, ad
        torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    line = json.dumps(result)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
