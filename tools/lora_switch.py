"""What switching a LoRA costs on the SDXL UNet, against the only alternative without device-side merging:

    (a) a rank-16 adapter on the attention projections, (b) a rank-64 adapter on every weight of two or more dimensions

    python tools/lora_switch.py [--switches 20] [--nfe 50] [--out FILE]

Per adapter: the time of `set_lora_scales` (merge from the pristine copy + every refreshed packed layout) by CUDA events
on the current stream, after two untimed switches, alternating between two scales; median, min and max of the
switches; `bytes_moved` (from shapes) over that time against the data-sheet 3.35 TB/s of HBM3 (the job is HBM-bound: its
least time is bytes over bandwidth, the tensor-core work is far below it). The alternative, building a new engine from a
host-merged state dict, is timed once with the host clock around work that ends in a device synchronise (merge on the
host in fp32 excluded: only the upload, the repack and the plan). `ddim_cfg++` at 1024^2, batch 2, runs with and
without adapter (a): same plan, so the same speed is expected, and measured. The GPU's name, power limit and max SM
clock are read in the same process, before and after. Needs a CUDA device; there is no fallback."""
from __future__ import annotations

import argparse
import json
import math
import statistics
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.batch_throughput import gpu_info  # noqa: E402
from tools.refiner_throughput import conditioning, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # NVIDIA data sheet, H100 SXM HBM3


def make_adapter(cfg, rank: int, pick, seed: int):
    from cfgpp_b200 import weights as Wt
    from cfgpp_b200.lora import LoraAdapter
    g = torch.Generator(device="cuda").manual_seed(seed)
    targets = {}
    for key, shape, _ in Wt.unet_param_specs(cfg):
        if len(shape) < 2 or not pick(key):
            continue
        N, K = shape[0], math.prod(shape[1:])
        down = (torch.randn(rank, K, generator=g, device="cuda") / math.sqrt(K)).half()
        up = (torch.randn(N, rank, generator=g, device="cuda") * (0.1 / math.sqrt(rank))).half()
        targets[key] = (down, up, float(rank))
    return LoraAdapter(targets)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--switches", type=int, default=20)
    ap.add_argument("--nfe", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3, help="timed trajectories with and without the adapter, alternating")
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_switch.py measures on a CUDA device; none is visible")
    from cfgpp_b200 import config as C, schedule as S, weights as Wt
    from cfgpp_b200.engine import NativeUNet

    cfg = C.sdxl_config()
    dev = torch.device("cuda:0")
    result = {"gpu": gpu_info(), "model": "sdxl", "switches": args.switches, "hbm_data_sheet_bytes_per_s": HBM_BYTES_PER_S,
              "timing": "CUDA events around set_lora_scales after two warm-up switches, scales alternating; rebuild: "
                        "host clock around NativeUNet(...) + prepare, ending in a device synchronise"}
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    t0 = time.perf_counter()
    eng = NativeUNet(cfg, sd, dev)
    eng.prepare(2, 128, 128)
    torch.cuda.synchronize()
    result["rebuild_handle_s"] = time.perf_counter() - t0
    print(f"new handle from a state dict on the device (upload, repack, plan): {result['rebuild_handle_s']:.2f} s", flush=True)

    B, hw, lam = 2, 128, 0.6
    g = torch.Generator().manual_seed(0)
    zT = torch.randn(B, 4, hw, hw, generator=g)
    uc, c, add = conditioning(cfg, B, g, [(1024., 1024.)] * (2 * B))
    steps = S.ddim_cfgpp_steps(S.Schedule.make(args.nfe), lam, sdxl_indexing=True)

    def trajectory():
        eng.set_state(zT)
        eng.run_steps(0, len(steps))

    def bind():
        eng.bind_prompt(uc, c, add["text_embeds"], add["time_ids"], force=True)
        eng.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)

    cases = (("attention_rank16", 16, lambda k: ".attn" in k and ".to_" in k),
             ("every_weight_rank64", 64, lambda k: True))
    for label, rank, pick in cases:
        ad = make_adapter(cfg, rank, pick, seed=rank)
        name = eng.add_lora(ad, 0.8, name=label)
        for s in (0.6, 0.8):
            eng.set_lora_scales({name: s})
        torch.cuda.synchronize()
        ms = [timed(lambda s=s: eng.set_lora_scales({name: s})) for s in [0.6, 0.8] * (args.switches // 2)]
        st = eng.lora_stats
        med = statistics.median(ms)
        row = {"rank": rank, "targets": st["targets"], "backup_bytes": st["backup_bytes"], "bytes_moved": st["bytes_moved"],
               "ms_median": med, "ms_min": min(ms), "ms_max": max(ms),
               "bytes_per_s_median": st["bytes_moved"] / med * 1e3,
               "share_of_hbm_data_sheet": st["bytes_moved"] / med * 1e3 / HBM_BYTES_PER_S}
        print(f"{label}: {st['targets']} targets, backup {st['backup_bytes'] / 2**30:.2f} GiB, moves "
              f"{st['bytes_moved'] / 1e9:.2f} GB in {med:.2f} ms median [{min(ms):.2f}, {max(ms):.2f}] = "
              f"{row['bytes_per_s_median'] / 1e12:.2f} TB/s ({100 * row['share_of_hbm_data_sheet']:.0f}% of the HBM3 data "
              f"sheet, HBM-bound)", flush=True)
        if label == "attention_rank16":
            with_ms, without_ms = [], []
            for _ in range(args.reps):
                eng.set_lora_scales({name: 0.8})
                bind(); trajectory()
                with_ms.append(timed(trajectory))
                eng.set_lora_scales({name: 0.0})
                bind(); trajectory()
                without_ms.append(timed(trajectory))
            row["images_per_s_with"] = B / min(with_ms) * 1e3
            row["images_per_s_scale0"] = B / min(without_ms) * 1e3
            print(f"ddim_cfg++ NFE {args.nfe}, 1024^2, batch {B}: {row['images_per_s_with']:.3f} img/s with the adapter, "
                  f"{row['images_per_s_scale0']:.3f} img/s at scale 0", flush=True)
        result[label] = row
        eng.clear_lora()
    bind(); trajectory()
    base_ms = min(timed(trajectory) for _ in range(args.reps))
    result["images_per_s_no_adapter"] = B / base_ms * 1e3
    print(f"no adapter loaded: {result['images_per_s_no_adapter']:.3f} img/s", flush=True)
    result["gpu_after"] = gpu_info()
    line = json.dumps(result)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
