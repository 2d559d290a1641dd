"""Time the native flash-attention kernel at every distinct attention shape of the UNets' transformer blocks, beside
torch's scaled_dot_product_attention (cuDNN and flash backends) on the same card.

    python tools/attention_bench.py [--batches 4 16] [--rounds 5] [--iters 50] [--out FILE]

Shapes: `tests/production.py::unet_attn_launches` for SDXL 1024², SD 2 768² and SD v1.5 512² at UNet batch 4 and 16,
each distinct (heads, Nq, Nkv, head_dim) once. The native kernel reads q / k / v in the UNet's layouts: column slices of
the fused [NB, N, 3·H·P] QKV buffer for self-attention, q from its own buffer and k / v slices of the [NB, 77, 2·H·P]
KV buffer for cross-attention (P = head_dim padded to 64). SDPA runs on contiguous [NB, H, N, P] tensors.

Per shape: µs per launch from CUDA events around `--iters` back-to-back launches after warm-up, median (min, max) of
`--rounds` rounds; algorithmic TFLOP/s (4·NB·H·Nq·Nkv·head_dim / time); and that rate as a fraction of the 989 TFLOP/s
dense FP16 data-sheet figure of the H100 SXM (a reference line, not a reached rate). The card's name, power limit and
maximum SM clock are read in the same process (`nvidia-smi`, read-only), and the library path is printed so that one
run can compare two builds through CFGPP_B200_LIB. Needs a CUDA GPU; the shape table is printed before that check."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

DATASHEET_TFLOPS = 989.0
MODELS = (("sdxl", 128, 128), ("sd2", 96, 96), ("sd15", 64, 64))


def shapes(batches):
    """[(tag, NB, heads, Nq, Nkv, head_dim, flops)], each distinct shape once per batch."""
    import production as P
    from cfgpp_b200 import config as C
    out, seen = [], set()
    for NB in batches:
        for m, h, w in MODELS:
            for l in P.unet_attn_launches(C.CONFIGS[m](), h, w, NB=NB):
                key = (NB, l["heads"], l["Nq"], l["Nkv"], l["hd"])
                if key in seen:
                    continue
                seen.add(key)
                kind = "self" if l["Nq"] == l["Nkv"] else "cross"
                out.append((f"{P.size_tag(m, h, w)}-{kind}", *key, l["flops"]))
    return out


def time_us(fn, iters, rounds):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        per.append(a.elapsed_time(b) * 1e3 / iters)
    return statistics.median(per), min(per), max(per)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 16])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", type=str, default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    table = shapes(args.batches)
    for tag, NB, H, Nq, Nkv, hd, fl in table:
        print(f"shape {tag} NB{NB} H{H} {Nq}x{Nkv} hd{hd}: {fl / 1e9:.2f} GFLOP")

    import torch
    if not torch.cuda.is_available():
        sys.exit("attention_bench: needs a CUDA GPU")
    from torch.nn.attention import SDPBackend, sdpa_kernel
    import torch.nn.functional as F
    from cfgpp_b200 import _native as nv

    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    card = smi[0] if smi else torch.cuda.get_device_name(0)
    header = {"card": card, "lib": str(nv.lib_path()), "datasheet_tflops": DATASHEET_TFLOPS}
    print(json.dumps(header))
    lines = [header]
    backends = (("cudnn", SDPBackend.CUDNN_ATTENTION), ("flash", SDPBackend.FLASH_ATTENTION))
    g = torch.Generator(device=dev).manual_seed(0)
    for tag, NB, H, Nq, Nkv, hd, fl in table:
        P = (hd + 63) // 64 * 64
        C = H * P
        if Nq == Nkv:
            qkv = torch.randn(NB, Nq, 3 * C, generator=g, device=dev).half()
            q, k, v = qkv[:, :, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:]
        else:
            q = torch.randn(NB, Nq, C, generator=g, device=dev).half()
            kv = torch.randn(NB, Nkv, 2 * C, generator=g, device=dev).half()
            k, v = kv[:, :, :C], kv[:, :, C:]
        rec = {"shape": tag, "NB": NB, "heads": H, "Nq": Nq, "Nkv": Nkv, "head_dim": hd, "gflop": fl / 1e9}
        med, lo, hi = time_us(lambda: nv.op_attention(q, k, v, H, head_dim=hd), args.iters, args.rounds)
        rec["native"] = {"us": med, "us_min": lo, "us_max": hi, "tflops": fl / med / 1e6,
                         "of_datasheet": fl / med / 1e6 / DATASHEET_TFLOPS}
        del q, k, v
        qs, ks, vs = (torch.randn(NB, H, n, P, generator=g, device=dev).half() for n in (Nq, Nkv, Nkv))
        for name, be in backends:
            try:
                with sdpa_kernel(be):
                    med, lo, hi = time_us(lambda: F.scaled_dot_product_attention(qs, ks, vs), args.iters,
                                          args.rounds)
                rec[f"sdpa_{name}"] = {"us": med, "us_min": lo, "us_max": hi, "tflops": fl / med / 1e6}
            except RuntimeError as e:
                rec[f"sdpa_{name}"] = {"did_not_run": str(e).splitlines()[0][:160]}
        del qs, ks, vs
        print(json.dumps(rec))
        lines.append(rec)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
