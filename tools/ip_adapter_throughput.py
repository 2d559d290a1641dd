"""The fused step with and without an IP-Adapter, at SD v1.5 512^2 batch 4 and SDXL 1024^2 batch 2:

    python tools/ip_adapter_throughput.py [--nfe 50] [--reps 3] [--out FILE]

Per configuration one engine on seeded synthetic weights runs a `ddim_cfg++` trajectory of NFE fused steps, without
an adapter and with a synthetic one (4 image tokens, E = 1024 / 1280) attached at scale 1; the two alternate over
`reps` timed trajectories (CUDA events around the NFE graph replays alone, after one warm-up trajectory of each side).
The vision tower's time per image is the best of 5 encodes at batch 1 and 8. Then, per side, ten eager profiled forwards (`profile_forward`, CUDA events around every plan entry) give the summed
time of the `attn2.sdpa` launches, best of ten. The once-per-image projections are not a step cost and are not timed.
The GPU's name, power limit and max SM clock are read in the same process, before and after. Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.batch_throughput import gpu_info  # noqa: E402
from tools.refiner_throughput import timed  # noqa: E402

CONFIGS = (("sd15", 4, 64, 1024), ("sdxl", 2, 128, 1280))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nfe", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3, help="timed trajectories of each side, alternating")
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ip_adapter_throughput.py measures on a CUDA device; none is visible")
    from cfgpp_b200 import config as C, ip_adapter as IP, schedule as S, weights as Wt
    from cfgpp_b200.engine import NativeUNet

    result = {"gpu": gpu_info(), "method": "ddim_cfg++", "nfe": args.nfe, "reps": args.reps,
              "timing": "CUDA events around NFE fused steps (run_steps), after one warm-up trajectory each; without "
                        "and with the adapter alternate. attn2_ms: summed attn2.sdpa launches of one profiled eager "
                        "forward, best of 10", "configs": []}
    for name, B, hw, E in CONFIGS:
        cfg = C.CONFIGS[name]()
        eng = NativeUNet(cfg, Wt.synthetic_state_dict(cfg, seed=1234, device="cuda"), "cuda:0")
        ad = IP.IPAdapter(f"ip-{name}", "cuda:0", cfg)
        g = torch.Generator().manual_seed(0)
        zT = torch.randn(B, 4, hw, hw, generator=g).cuda()
        uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
        c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().cuda()
        pooled = tids = None
        if cfg.addition_embed_type == "text_time":
            pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().cuda()
            tids = torch.tensor([[8. * hw, 8. * hw, 0, 0, 8. * hw, 8. * hw]] * (2 * B)).cuda()
        embeds = torch.randn(B, E, generator=g).half().cuda()
        steps = S.ddim_cfgpp_steps(S.Schedule.make(args.nfe), 0.6, sdxl_indexing=cfg.addition_embed_type is not None)

        def setup(adapter: bool):
            eng.attach_ip_adapter(ad if adapter else None)
            eng.prepare(B, hw, hw)
            eng.bind_prompt(uc, c, pooled, tids, force=True)
            if adapter:
                eng.set_ip_image_embeds(embeds)
            eng.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
            stats = dict(eng.plan_stats, launches_per_step=eng.launches_per_step)

            def traj():
                eng.run_steps(0, len(steps))
            eng.set_state(zT)
            traj()  # warm-up: captures the step graph
            torch.cuda.synchronize()
            return stats, traj

        sides, times, attn2 = {}, {False: [], True: []}, {}
        for _ in range(args.reps):
            for adapter in (False, True):
                stats, traj = setup(adapter)
                sides[adapter] = stats
                eng.set_state(zT)
                times[adapter].append(timed(traj) / len(steps))
                if adapter not in attn2:
                    attn2[adapter] = min(sum(ms for n, _, _, ms in eng.profile_forward(zT, 500.0)
                                             if n.endswith("attn2.sdpa")) for _ in range(10))
        assert torch.isfinite(eng.get_state(0)).all()
        row = {"model": name, "batch": B, "resolution": [8 * hw, 8 * hw], "image_embed_dim": E, "ip_tokens": 4}
        for adapter, label in ((False, "plain"), (True, "ip_adapter")):
            st = sides[adapter]
            row[label] = {"ms_per_step": times[adapter], "ms_per_step_best": min(times[adapter]),
                          "step_flops": st["step_flops"], "launches_per_step": st["launches_per_step"],
                          "attn2_ms": attn2[adapter]}
        px = torch.randn(8, 3, 224, 224, generator=g).cuda()
        ad.encoder.encode(px)  # warm-up at the timed batch
        row["vision_tower"] = {"config": f"{ad.encoder_cfg.hidden_size}x{ad.encoder_cfg.num_hidden_layers}",
                               "ms_per_image_b1": min(timed(lambda: ad.encoder.encode(px[:1])) for _ in range(5)),
                               "ms_per_image_b8": min(timed(lambda: ad.encoder.encode(px)) for _ in range(5)) / 8}
        ad.close()
        row["step_ratio"] = row["ip_adapter"]["ms_per_step_best"] / row["plain"]["ms_per_step_best"]
        print(f"{name} B={B} {8 * hw}^2: plain {row['plain']['ms_per_step_best']:.2f} ms/step "
              f"(attn2 {attn2[False]:.3f} ms), IP-Adapter {row['ip_adapter']['ms_per_step_best']:.2f} ms/step "
              f"(attn2 {attn2[True]:.3f} ms); step time ratio {row['step_ratio']:.4f}; vision tower "
              f"{row['vision_tower']}", flush=True)
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
