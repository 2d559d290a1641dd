"""The fused step with no adapter, the plain IP-Adapter (4 image tokens) and IP-Adapter Plus (16 tokens), at SD v1.5
512^2 batch 4 and SDXL 1024^2 batch 2; the Resampler per call; the vision tower's hidden-state output per image:

    python tools/ip_adapter_plus_throughput.py [--nfe 50] [--reps 3] [--out FILE]

Per configuration one engine on seeded synthetic weights runs a `ddim_cfg++` trajectory of NFE fused steps; the three
sides alternate over `reps` timed trajectories (CUDA events around the NFE graph replays alone, after one warm-up
trajectory of each). At UNet batch NB = 2 and 16, the Resampler alone (the plan's `image_proj.*` entries, through the
measurement entry point `cfgpp_dbg_ip_image_proj`, on the hidden states already set) is timed as the mean of 20 calls,
best of 5, and `set_ip_image_embeds` of the Plus adapter (host row assembly, the Resampler and every block's image
K / V projection: once per reference image) as the best of 5; the vision
tower's `encode_hidden` (ViT-H/14, penultimate layer) per image is the best of 5 at batch 1 and 8. The GPU's name,
power limit and max SM clock are read in the same process, before and after. Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.batch_throughput import gpu_info  # noqa: E402
from tools.refiner_throughput import timed  # noqa: E402

CONFIGS = (("sd15", 4, 64), ("sdxl", 2, 128))
SIDES = ("none", "plain", "plus")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nfe", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3, help="timed trajectories of each side, alternating")
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ip_adapter_plus_throughput.py measures on a CUDA device; none is visible")
    from cfgpp_b200 import config as C, ip_adapter as IP, schedule as S, weights as Wt
    from cfgpp_b200.engine import NativeUNet

    result = {"gpu": gpu_info(), "method": "ddim_cfg++", "nfe": args.nfe, "reps": args.reps,
              "timing": "CUDA events around NFE fused steps (run_steps), after one warm-up trajectory each; no "
                        "adapter, plain and Plus alternate. resampler_ms: the image_proj.* plan entries alone, "
                        "mean of 20 calls, best of 5; set_embeds_ms: set_ip_image_embeds of the Plus adapter (Resampler "
                        "+ image K/V projections + host row assembly), best of 5", "configs": []}
    for name, B, hw in CONFIGS:
        cfg = C.CONFIGS[name]()
        eng = NativeUNet(cfg, Wt.synthetic_state_dict(cfg, seed=1234, device="cuda"), "cuda:0")
        ads = {"none": None, "plain": IP.IPAdapter(f"ip-{name}", "cuda:0", cfg),
               "plus": IP.IPAdapter(f"plus-{name}", "cuda:0", cfg, image_proj="resampler")}
        g = torch.Generator().manual_seed(0)
        zT = torch.randn(B, 4, hw, hw, generator=g).cuda()
        uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
        c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
        pooled = tids = None
        if cfg.addition_embed_type == "text_time":
            pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().cuda()
            tids = torch.tensor([[8. * hw, 8. * hw, 0, 0, 8. * hw, 8. * hw]] * (2 * B)).cuda()
        plus = ads["plus"]
        plus._uncond = torch.randn(1, plus.resampler["seq_len"], plus.embed_dim, generator=g).half().cuda()
        embeds = {"plain": torch.randn(B, ads["plain"].embed_dim, generator=g).half().cuda(),
                  "plus": torch.randn(B, plus.resampler["seq_len"], plus.embed_dim, generator=g).half().cuda()}
        steps = S.ddim_cfgpp_steps(S.Schedule.make(args.nfe), 0.6, sdxl_indexing=cfg.addition_embed_type is not None)

        def bind(side: str, batch: int):
            """prepare for `batch` images, the first image's prompt (and Plus image) repeated"""
            eng.attach_ip_adapter(ads[side])
            eng.prepare(batch, hw, hw)
            eng.bind_prompt(uc[:1].repeat(batch, 1, 1), c[:1].repeat(batch, 1, 1),
                            None if pooled is None else pooled[:1].repeat(2 * batch, 1),
                            None if tids is None else tids[:1].repeat(2 * batch, 1), force=True)

        def trajectory(side: str):
            eng.attach_ip_adapter(ads[side])
            eng.prepare(B, hw, hw)
            eng.bind_prompt(uc, c, pooled, tids, force=True)
            if side != "none":
                eng.set_ip_image_embeds(embeds[side])
            eng.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
            stats = dict(eng.plan_stats, launches_per_step=eng.launches_per_step)

            def traj():
                eng.run_steps(0, len(steps))
            eng.set_state(zT)
            traj()  # warm-up: captures the step graph
            torch.cuda.synchronize()
            return stats, traj

        stats, times = {}, {s: [] for s in SIDES}
        for _ in range(args.reps):
            for side in SIDES:
                stats[side], traj = trajectory(side)
                eng.set_state(zT)
                times[side].append(timed(traj) / len(steps))
        assert torch.isfinite(eng.get_state(0)).all()
        row = {"model": name, "batch": B, "resolution": [8 * hw, 8 * hw], "plus": plus.resampler}
        for side in SIDES:
            row[side] = {"ms_per_step": times[side], "ms_per_step_best": min(times[side]),
                         "step_flops": stats[side]["step_flops"], "launches_per_step": stats[side]["launches_per_step"]}
        row["resampler_ms"], row["set_embeds_ms"] = {}, {}
        from cfgpp_b200 import _native as nv

        def resampler():
            nv.check(eng.lib.cfgpp_dbg_ip_image_proj(eng._h, None, nv.stream_ptr()))
        for NB in (2, 16):
            bind("plus", NB // 2)
            e = embeds["plus"][:1].repeat(NB // 2, 1, 1)
            eng.set_ip_image_embeds(e)
            row["set_embeds_ms"][f"NB{NB}"] = min(timed(lambda: eng.set_ip_image_embeds(e)) for _ in range(5))
            row["resampler_ms"][f"NB{NB}"] = min(timed(resampler, 20) / 20 for _ in range(5))
        px = torch.randn(8, 3, 224, 224, generator=g).cuda()
        enc = plus.encoder
        enc.encode_hidden(px)
        enc.encode_hidden(px[:1])
        row["encode_hidden"] = {"config": f"{plus.encoder_cfg.hidden_size}x{plus.encoder_cfg.num_hidden_layers}",
                                "ms_per_image_b1": min(timed(lambda: enc.encode_hidden(px[:1])) for _ in range(5)),
                                "ms_per_image_b8": min(timed(lambda: enc.encode_hidden(px)) for _ in range(5)) / 8}
        for ad in ads.values():
            if ad is not None:
                ad.close()
        print(f"{name} B={B} {8 * hw}^2: " + ", ".join(f"{s} {row[s]['ms_per_step_best']:.3f} ms/step" for s in SIDES)
              + f"; Resampler {row['resampler_ms']}; set_ip_image_embeds {row['set_embeds_ms']}; encode_hidden {row['encode_hidden']}", flush=True)
        result["configs"].append(row)
        eng.close()
        del eng
        torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    line = json.dumps(result)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
