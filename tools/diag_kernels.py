"""GPU diagnostic sweep of the operator-level kernels against torch references (needs a GPU).

Prints one line per case and never aborts on a mismatch, so that a single GPU call yields the full picture.
    python tools/diag_kernels.py [gemm] [conv] [attn] [norm] ...
"""
from __future__ import annotations

import sys
import time
import traceback
from pathlib import Path

import os
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from cfgpp_b200 import _native as nv  # noqa: E402

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda:0")
RESULTS = []


def report(name, got, ref, tol=2e-3):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    denom = ref.abs().max().item() + 1e-12
    rel = err.max().item() / denom
    relL2 = (got - ref).norm().item() / (ref.norm().item() + 1e-12)
    ok = bool(torch.isfinite(got).all()) and relL2 < tol
    line = f"[{'OK ' if ok else 'BAD'}] {name}: relL2={relL2:.3e} maxerr/max={rel:.3e} max|ref|={denom:.3f}"
    print(line, flush=True)
    if not ok:
        # error structure: which 8-row / 8-col residues are wrong (swizzle / descriptor diagnosis)
        e2 = err.reshape(-1, err.shape[-1])
        bad = e2 > (0.02 * denom)
        print(f"      bad frac={bad.float().mean().item():.4f}  rows bad (first 16 of {e2.shape[0]}): "
              f"{bad.any(1)[:16].int().tolist()}  cols bad (first 32): {bad.any(0)[:32].int().tolist()}")
        rb = bad.any(1).reshape(-1).cpu()
        cb = bad.any(0).reshape(-1).cpu()
        ridx = torch.arange(rb.numel())
        print(f"      bad rows by (row%128)//32: {[int(rb[(ridx % 128) // 32 == i].sum()) for i in range(4)]}"
              f"  by row%8: {[int(rb[ridx % 8 == i].sum()) for i in range(8)]}")
        cidx = torch.arange(cb.numel())
        print(f"      bad cols by (col%64)//8: {[int(cb[(cidx % 64) // 8 == i].sum()) for i in range(8)]}"
              f"  by col//32 (first 8): {[int(cb[32*i:32*i+32].sum()) for i in range(min(8, cb.numel() // 32))]}")
        print(f"      got[0,:8]={got.reshape(-1, got.shape[-1])[0, :8].tolist()}")
        print(f"      ref[0,:8]={ref.reshape(-1, ref.shape[-1])[0, :8].tolist()}")
    RESULTS.append((name, ok))
    return ok


def guarded(name, fn):
    try:
        fn()
        torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        print(f"[EXC] {name}: {type(e).__name__}: {e}", flush=True)
        traceback.print_exc()
        RESULTS.append((name, False))


def ref_linear(a, w, bias, addend, rows_per_group):
    acc = a.float() @ w.float().t()
    if bias is not None:
        acc = acc + bias.float()
    t = acc.half()
    if addend is not None:
        ad = addend.float()
        if rows_per_group > 1:
            ad = ad.repeat_interleave(rows_per_group, dim=0)[: a.shape[0]]
        t = (t.float() + ad).half()
    return t


def diag_gemm():
    g = torch.Generator(device="cpu").manual_seed(0)

    def rnd(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).half().to(dev)

    cases = [
        # M, N, K, bias, addend(0 none / 1 full / >1 rows-per-group), force_bn
        (128, 64, 64, False, 0, 64),
        (128, 128, 64, False, 0, 128),
        (128, 128, 128, False, 0, 128),
        (256, 256, 256, True, 0, 256),
        (256, 320, 320, True, 1, 160),
        (308, 1280, 2048, False, 0, 0),
        (4096, 1280, 1280, True, 1, 0),
        (4096, 640, 640, True, 1, 0),
        (2048, 320, 960, True, 1024, 0),
        (1000, 200, 192, True, 1, 128),
        (16384, 1920, 640, False, 0, 0),
        (4096, 1280, 5120, True, 1, 0),
    ]
    for (M, N, K, hb, ha, bn) in cases:
        name = f"linear M={M} N={N} K={K} bias={hb} add={ha} bn={bn}"

        def run():
            a = rnd(M, K)
            w = rnd(N, K, scale=K ** -0.5)
            bias = rnd(N) if hb else None
            addend = None
            if ha == 1:
                addend = rnd(M, N)
            elif ha > 1:
                addend = rnd((M + ha - 1) // ha, N)
            out = nv.op_linear(a, w, bias, addend, ha if ha > 1 else 1, force_bn=bn)
            report(name, out, ref_linear(a, w, bias, addend, ha))

        guarded(name, run)

    # dual-source A (K concat)
    def run_dual():
        M, K1, K2, N = 1024, 640, 320, 320
        a1, a2 = rnd(M, K1), rnd(M, K2)
        w = rnd(N, K1 + K2, scale=(K1 + K2) ** -0.5)
        bias = rnd(N)
        out = nv.op_linear(a1, w, bias, None, 1, a2=a2)
        report("linear dual-source", out, ref_linear(torch.cat([a1, a2], 1), w, bias, None, 1))

    guarded("linear dual-source", run_dual)

    # GEGLU: weight rows interleaved per 256-row tile as 128 value + 128 gate
    def run_geglu():
        M, C = 512, 640
        inner = 4 * C
        a = rnd(M, C)
        w = rnd(2 * inner, C, scale=C ** -0.5)  # torch layout: rows [0,inner) value, [inner, 2 inner) gate
        b = rnd(2 * inner)
        idx = []
        for t in range(inner // 128):
            idx += list(range(t * 128, t * 128 + 128)) + list(range(inner + t * 128, inner + t * 128 + 128))
        idx = torch.tensor(idx, device=dev)
        out = nv.op_linear(a, w[idx].contiguous(), b[idx].contiguous(), geglu=True)
        h = (a.float() @ w.float().t() + b.float()).half()
        val, gate = h[:, :inner], h[:, inner:]
        ref = (val.float() * torch.nn.functional.gelu(gate.float()).half().float()).half()
        report("linear GEGLU", out, ref)

    guarded("linear GEGLU", run_geglu)


def diag_conv():
    g = torch.Generator(device="cpu").manual_seed(1)

    def rnd(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).half().to(dev)

    cases = [
        # B, H, W, Cin, Cout, bias, temb, residual, bn
        (1, 32, 32, 64, 64, False, False, False, 64),
        (2, 32, 32, 64, 128, True, False, False, 128),
        (1, 128, 128, 64, 64, False, False, False, 64),
        (2, 64, 64, 128, 128, True, True, False, 0),
        (4, 16, 16, 128, 256, True, False, True, 0),
        (2, 8, 8, 128, 128, True, True, False, 0),
        (1, 128, 128, 320, 320, True, True, False, 0),
        (2, 64, 64, 640, 320, True, False, True, 0),
        (4, 32, 32, 1280, 1280, True, True, False, 0),
    ]
    for (B, H, W, Cin, Cout, hb, ht, hr, bn) in cases:
        name = f"conv3x3 B={B} H={H} W={W} Cin={Cin} Cout={Cout} bias={hb} temb={ht} res={hr} bn={bn}"

        def run():
            x = rnd(B, Cin, H, W)
            w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
            bias = rnd(Cout) if hb else None
            x_nhwc = x.permute(0, 2, 3, 1).contiguous()
            w_packed = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
            addend, rpg = None, 1
            if ht:
                addend, rpg = rnd(B, Cout), H * W
            elif hr:
                addend = rnd(B * H * W, Cout)
            out = nv.op_conv3x3(x_nhwc, w_packed, bias, addend, rpg)
            ref = torch.nn.functional.conv2d(x.float(), w.float(), bias.float() if hb else None, padding=1)
            ref = ref.half().permute(0, 2, 3, 1).reshape(B * H * W, Cout)
            if ht:
                ref = (ref.float() + addend.float().repeat_interleave(H * W, 0)).half()
            elif hr:
                ref = (ref.float() + addend.float()).half()
            report(name, out.reshape(B * H * W, Cout), ref)

        guarded(name, run)


def bench_gemm():
    print("--- GEMM timing (CUDA events, 20 iters) ---", flush=True)
    g = torch.Generator(device="cpu").manual_seed(2)
    shapes = [(4096, 1280, 1280, 0), (4096, 3840, 1280, 0), (4096, 1280, 5120, 0), (16384, 640, 640, 0),
              (16384, 1920, 640, 0), (16384, 640, 2560, 0), (65536, 320, 320, 0), (8192, 8192, 8192, 256),
              (4096, 1280, 1280, 128), (4096, 1280, 1280, 160), (4096, 1280, 1280, 256)]
    for (M, N, K, bn) in shapes:
        try:
            a = (torch.randn(M, K, generator=g)).half().to(dev)
            w = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(dev)
            for _ in range(3):
                nv.op_linear(a, w, force_bn=bn)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                nv.op_linear(a, w, force_bn=bn)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 20
            e0.record()
            for _ in range(20):
                torch.matmul(a, w.t())
            e1.record()
            torch.cuda.synchronize()
            ms_t = e0.elapsed_time(e1) / 20
            tf = 2.0 * M * N * K / ms / 1e9
            print(f"gemm M={M} N={N} K={K} bn={bn}: {ms*1e3:.1f} us  {tf:.0f} TFLOP/s   (torch.matmul {ms_t*1e3:.1f} us "
                  f"{2.0*M*N*K/ms_t/1e9:.0f} TFLOP/s)", flush=True)
        except Exception as e:  # noqa: BLE001
            print(f"[EXC] bench gemm {M},{N},{K}: {e}", flush=True)

    print("--- conv3x3 timing ---", flush=True)
    for (B, H, W, Cin, Cout) in [(4, 128, 128, 320, 320), (4, 64, 64, 640, 640), (4, 32, 32, 1280, 1280),
                                 (4, 32, 32, 2560, 1280)]:
        try:
            x = torch.randn(B, Cin, H, W, generator=g).half().to(dev)
            w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).half().to(dev)
            x_nhwc = x.permute(0, 2, 3, 1).contiguous()
            w_packed = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
            xcl = x.contiguous(memory_format=torch.channels_last)
            wcl = w.contiguous(memory_format=torch.channels_last)
            for _ in range(3):
                nv.op_conv3x3(x_nhwc, w_packed)
                torch.nn.functional.conv2d(x, w, padding=1)
                torch.nn.functional.conv2d(xcl, wcl, padding=1)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            res = []
            for fn in (lambda: nv.op_conv3x3(x_nhwc, w_packed), lambda: torch.nn.functional.conv2d(x, w, padding=1),
                       lambda: torch.nn.functional.conv2d(xcl, wcl, padding=1)):
                e0.record()
                for _ in range(10):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                res.append(e0.elapsed_time(e1) / 10)
            fl = 2.0 * B * H * W * Cout * Cin * 9
            print(f"conv B={B} {H}x{W} {Cin}->{Cout}: ours {res[0]*1e3:.1f} us {fl/res[0]/1e9:.0f} TF/s | cudnn nchw "
                  f"{res[1]*1e3:.1f} us {fl/res[1]/1e9:.0f} | cudnn nhwc {res[2]*1e3:.1f} us {fl/res[2]/1e9:.0f}", flush=True)
        except Exception as e:  # noqa: BLE001
            print(f"[EXC] bench conv: {e}", flush=True)


def diag_attn():
    g = torch.Generator(device="cpu").manual_seed(3)
    cases = [(1, 1, 128, 128), (2, 2, 256, 256), (1, 4, 64, 64), (2, 5, 1024, 1024), (1, 10, 4096, 4096),
             (2, 4, 256, 77), (4, 20, 1024, 77), (1, 2, 200, 333)]
    for (B, H, Nq, Nkv) in cases:
        name = f"attention B={B} H={H} Nq={Nq} Nkv={Nkv}"

        def run():
            C = H * 64
            if Nq == Nkv:
                qkv = (torch.randn(B, Nq, 3 * C, generator=g) * 1.2).half().to(dev)
                q, k, v = qkv[:, :, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:]
            else:
                q = (torch.randn(B, Nq, C, generator=g) * 1.2).half().to(dev)
                kv = (torch.randn(B, Nkv, 2 * C, generator=g) * 1.2).half().to(dev)
                k, v = kv[:, :, :C], kv[:, :, C:]
            out = nv.op_attention(q, k, v, H)
            qf, kf, vf = (t.float().reshape(B, -1, H, 64).transpose(1, 2) for t in (q, k, v))
            ref = torch.nn.functional.scaled_dot_product_attention(qf, kf, vf)
            ref = ref.transpose(1, 2).reshape(B, Nq, C)
            report(name, out, ref, tol=3e-3)

        guarded(name, run)


def graph_time_us(fn, iters=40):
    """Per-call device time of `fn` (enqueues on the current stream) replayed inside one CUDA graph."""
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for _ in range(iters):
                fn()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / iters


def bench_gemm_graph():
    """Graph-timed GEMM / GEGLU / conv launches at the SDXL shapes (UNet batch 4)."""
    g = torch.Generator(device="cpu").manual_seed(2)
    for (M, N, K, geglu) in [(4096, 1280, 1280, False), (4096, 3840, 1280, False), (4096, 1280, 5120, False),
                             (4096, 10240, 1280, True), (16384, 640, 640, False), (16384, 1920, 640, False),
                             (16384, 640, 2560, False), (16384, 5120, 640, True), (4096, 1280, 2560, False),
                             (65536, 320, 960, False)]:
        a = torch.randn(M, K, generator=g).half().to(dev)
        w = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(dev)
        res = None if (geglu or os.environ.get('DIAG_NO_RES')) else torch.randn(M, N, generator=g).half().to(dev)
        bias = torch.randn(N, generator=g).half().to(dev)
        us = graph_time_us(lambda: nv.op_linear(a, w, bias, res, 1, geglu=geglu))
        print(f"gemm M={M} N={N} K={K} geglu={int(geglu)}: {us:7.1f} us  {2.0 * M * N * K / us / 1e6:6.0f} TFLOP/s", flush=True)
    for (B, H, W, Cin, Cout) in [(4, 128, 128, 320, 320), (4, 64, 64, 640, 640), (4, 32, 32, 1280, 1280),
                                 (4, 32, 32, 2560, 1280), (4, 64, 64, 1280, 640), (4, 128, 128, 640, 320)]:
        x = torch.randn(B, H, W, Cin, generator=g).half().to(dev)
        w = (torch.randn(Cout, 9 * Cin, generator=g) * (9 * Cin) ** -0.5).half().to(dev)
        bias = torch.randn(Cout, generator=g).half().to(dev)
        us = graph_time_us(lambda: nv.op_conv3x3(x, w, bias), iters=20)
        print(f"conv B={B} {H}x{W} {Cin}->{Cout}: {us:7.1f} us  {2.0 * B * H * W * Cout * Cin * 9 / us / 1e6:6.0f} TFLOP/s", flush=True)


def bench_attn():
    """Graph-timed attention launches at the SDXL / SD v1.5 shapes (batch 2 => UNet batch 4)."""
    g = torch.Generator(device="cpu").manual_seed(3)
    for (B, H, Nq, Nkv, hd) in [(4, 20, 1024, 1024, 64), (4, 10, 4096, 4096, 64), (4, 20, 1024, 77, 64),
                                (4, 10, 4096, 77, 64), (8, 8, 4096, 77, 40), (8, 8, 1024, 77, 80), (8, 8, 256, 77, 160),
                                (8, 8, 4096, 4096, 40), (8, 8, 1024, 1024, 80)]:
        P = (hd + 63) // 64 * 64
        C = H * P
        q = (torch.randn(B, Nq, C, generator=g) * 1.2).half().to(dev)
        k = (torch.randn(B, Nkv, C, generator=g) * 1.2).half().to(dev)
        v = (torch.randn(B, Nkv, C, generator=g) * 1.2).half().to(dev)
        us = graph_time_us(lambda: nv.op_attention(q, k, v, H, head_dim=hd))
        fl = 4.0 * B * H * Nq * Nkv * hd
        print(f"attention B={B} H={H} Nq={Nq} Nkv={Nkv} hd={hd}: {us:7.1f} us  {fl / us / 1e6:7.0f} TFLOP/s", flush=True)


def diag_norm():
    g = torch.Generator(device="cpu").manual_seed(4)

    def rnd(*s, scale=1.0, shift=0.0):
        return (torch.randn(*s, generator=g) * scale + shift).half().to(dev)

    for (B, HW, C1, C2, silu, eps) in [(2, 1024, 64, 0, True, 1e-5), (4, 16384, 320, 0, True, 1e-5),
                                       (2, 4096, 640, 320, True, 1e-5), (4, 1024, 1280, 1280, True, 1e-5),
                                       (2, 1024, 1280, 640, False, 1e-6), (2, 64, 256, 0, False, 1e-6)]:
        name = f"groupnorm B={B} HW={HW} C={C1}+{C2} silu={silu}"

        def run():
            x1 = rnd(B, HW, C1, scale=2.0, shift=0.5)
            x2 = rnd(B, HW, C2, scale=0.7, shift=-0.3) if C2 else None
            C = C1 + C2
            gamma, beta = rnd(C, scale=0.2, shift=1.0), rnd(C, scale=0.2)
            out = nv.op_groupnorm(x1, gamma, beta, eps, silu, x2)
            x = torch.cat([x1, x2], 2) if C2 else x1
            xn = x.float().permute(0, 2, 1).reshape(B, C, HW, 1)
            ref = torch.nn.functional.group_norm(xn, 32, gamma.float(), beta.float(), eps)
            if silu:
                ref = torch.nn.functional.silu(ref)
            ref = ref.reshape(B, C, HW).permute(0, 2, 1).half()
            report(name, out, ref, tol=1e-3)

        guarded(name, run)
    for (M, C) in [(4096, 1280), (16384, 640), (300, 128), (64, 256)]:
        name = f"layernorm M={M} C={C}"

        def run():
            x = rnd(M, C, scale=3.0, shift=1.0)
            gamma, beta = rnd(C, scale=0.2, shift=1.0), rnd(C, scale=0.2)
            out = nv.op_layernorm(x, gamma, beta)
            ref = torch.nn.functional.layer_norm(x.float(), (C,), gamma.float(), beta.float(), 1e-5).half()
            report(name, out, ref, tol=1e-3)

        guarded(name, run)


def _oracle_cfg(cfg):
    import dataclasses
    from oracle import unet as O
    return O.UNetConfig(**{f.name: getattr(cfg, f.name) for f in dataclasses.fields(O.UNetConfig)})


def _unet_inputs(cfg, B, hw, seed=7):
    g = torch.Generator(device="cpu").manual_seed(seed)
    z = torch.randn(B, 4, hw, hw, generator=g).to(dev)
    uc = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    c = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    add = None
    if cfg.addition_embed_type == "text_time":
        pooled = torch.randn(2 * B, cfg.pooled_dim, generator=g).half().to(dev)
        tid = torch.tensor([[hw * 8, hw * 8, 0, 0, hw * 8, hw * 8]] * (2 * B), dtype=torch.float16).to(dev)
        add = {"text_embeds": pooled, "time_ids": tid}
    return z, uc, c, add


def diag_unet(which=("tiny_sdxl", "tiny_sd15")):
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    from oracle import unet as O
    for name, B, hw, t in [("tiny_sdxl", 2, 32, 801), ("tiny_sd15", 1, 32, 401), ("tiny_sdxl", 1, 64, 21),
                           ("sdxl", 1, 128, 501), ("sd15", 1, 64, 401), ("sd15", 2, 64, 981)]:
        if name not in which:
            continue
        label = f"unet {name} B={B} latent={hw} t={t}"

        def run():
            cfg = C.CONFIGS[name]()
            sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
            z, uc, c, add = _unet_inputs(cfg, B, hw)
            net = NativeUNet(cfg, sd, dev)
            net.prepare(B, hw, hw)
            print(f"      workspace {net.workspace_bytes/2**20:.0f} MiB, forward {net.forward_flops/1e12:.3f} TFLOP, "
                  f"{net.launches_per_step} launches/step", flush=True)
            net.set_prompt(torch.cat([uc, c]), add["text_embeds"] if add else None,
                           add["time_ids"].float() if add else None)
            eu, ec = net.predict_noise(z, float(t))
            torch.cuda.synchronize()
            ocfg = _oracle_cfg(cfg)
            z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(t, device=dev), torch.cat([uc, c])
            m16 = O.build_unet(ocfg, sd, dtype=torch.float16, device=dev)
            with torch.autocast("cuda", dtype=torch.float16):
                r16 = m16(z_in, t_in, ctx, add)["sample"]
            del m16
            m32 = O.build_unet(ocfg, sd, dtype=torch.float32, device=dev)
            r32 = m32(z_in, t_in, ctx.float(), {k: v.float() for k, v in add.items()} if add else None)["sample"]
            del m32
            got = torch.cat([eu, ec]).float()
            e_ref = (r16.float() - r32).norm().item() / r32.norm().item()
            e_got = (got - r32).norm().item() / r32.norm().item()
            print(f"      std(eps)={r32.std().item():.4f}  relL2(ref16 vs fp32)={e_ref:.3e}  relL2(native vs fp32)={e_got:.3e}",
                  flush=True)
            report(label + " vs fp16-autocast oracle", got, r16, tol=5e-3)
            net.close()

        guarded(label, run)


def prof_unet(name="sdxl", B=2, hw=128):
    """Per-plan-entry CUDA-event profile of one eager forward (SDXL batch 2 by default), aggregated by op type."""
    import collections
    import re
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg = C.CONFIGS[name]()
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    z, uc, c, add = _unet_inputs(cfg, B, hw)
    net = NativeUNet(cfg, sd, dev)
    del sd
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"] if add else None, add["time_ids"].float() if add else None)
    net.profile_forward(z, 500.0)
    prof = net.profile_forward(z, 500.0)
    agg = collections.defaultdict(lambda: [0, 0.0, 0.0])
    for name, kind, fl, ms in prof:
        lvl = "L?"
        m = re.match(r"(down_blocks|up_blocks)\.(\d)", name)
        if m:
            i = int(m.group(2))
            top = len(cfg.block_out_channels) - 1
            lvl = f"L{i}" if m.group(1) == "down_blocks" else f"L{top - i}"
        elif name.startswith("mid_block"):
            lvl = f"L{len(cfg.block_out_channels) - 1}"
        short = re.sub(r"^.*?(resnets|attentions|downsamplers|upsamplers)\.\d+\.", "", name)
        short = re.sub(r"transformer_blocks\.\d+\.", "", short)
        key = (lvl, short, kind)
        agg[key][0] += 1
        agg[key][1] += ms
        agg[key][2] += fl
    tot = sum(v[1] for v in agg.values())
    print(f"total (eager, event-timed per entry) {tot:.2f} ms", flush=True)
    for (lvl, short, kind), (n, ms, fl) in sorted(agg.items(), key=lambda x: -x[1][1])[:40]:
        tf = fl / ms / 1e9 if ms > 0 and fl > 0 else 0
        print(f"  {ms:7.3f} ms {100*ms/tot:5.1f}%  n={n:3d} avg={1e3*ms/n:7.1f} us  {tf:6.0f} TF/s  {lvl} {short} kind={kind}", flush=True)
    bk = collections.defaultdict(lambda: [0.0, 0.0])
    for name, kind, fl, ms in prof:
        bk[kind][0] += ms
        bk[kind][1] += fl
    for k, nm in [(0, "linear"), (1, "conv3x3"), (2, "attention"), (3, "other")]:
        ms, fl = bk[k]
        print(f"  kind {nm}: {ms:.2f} ms  {fl/ms/1e9 if ms else 0:.0f} TF/s", flush=True)
    net.close()


def bench_unet():
    """First end-to-end timing of the SDXL step (B=2 -> UNet batch 4) vs the eager fp16-autocast oracle."""
    from cfgpp_b200 import config as C, weights as Wt, schedule as S
    from cfgpp_b200.engine import NativeUNet
    from oracle import unet as O
    cfg = C.sdxl_config()
    B, hw = 2, 128
    sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
    z, uc, c, add = _unet_inputs(cfg, B, hw)
    net = NativeUNet(cfg, sd, dev)
    net.prepare(B, hw, hw)
    net.set_prompt(torch.cat([uc, c]), add["text_embeds"], add["time_ids"].float())
    sch = S.Schedule.make(50)
    steps = S.ddim_cfgpp_steps(sch, 0.6, sdxl_indexing=True)
    net.set_schedule(S.STEP_DDIM_CFGPP, torch.float32, steps)
    net.set_state(z)
    net.run_steps(0, 3)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    net.run_steps(3, 10)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print(f"native fused step (graph): {ms:.2f} ms/step  -> {net.forward_flops/ms/1e9:.0f} TFLOP/s algorithmic, "
          f"{B/(50*ms/1e3):.3f} img/s @NFE=50", flush=True)
    for _ in range(2):
        net.predict_noise(z, 500.0)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(5):
        net.predict_noise(z, 500.0)
    e1.record()
    torch.cuda.synchronize()
    print(f"native eager forward: {e0.elapsed_time(e1)/5:.2f} ms", flush=True)
    net.close()
    del net
    m16 = O.build_unet(_oracle_cfg(cfg), sd, dtype=torch.float16, device=dev)
    z_in, t_in, ctx = torch.cat([z] * 2), torch.tensor(500, device=dev), torch.cat([uc, c])
    with torch.autocast("cuda", dtype=torch.float16), torch.no_grad():
        for _ in range(3):
            m16(z_in, t_in, ctx, add)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(5):
            m16(z_in, t_in, ctx, add)
        e1.record()
        torch.cuda.synchronize()
    print(f"eager torch fp16-autocast oracle forward: {e0.elapsed_time(e1)/5:.2f} ms", flush=True)


if __name__ == "__main__":
    which = set(sys.argv[1:]) or {"gemm", "conv", "bench"}
    t0 = time.time()
    print(f"device: {torch.cuda.get_device_name(0)}  lib: {nv.lib_path()}", flush=True)
    if "gemm" in which:
        diag_gemm()
    if "conv" in which:
        diag_conv()
    if "bench" in which:
        bench_gemm()
    if "attn" in which:
        diag_attn()
    if "norm" in which:
        diag_norm()
    if "bench_attn" in which:
        bench_attn()
    if "bench_gemm_graph" in which:
        bench_gemm_graph()
    if "unet_tiny" in which:
        diag_unet(("tiny_sdxl", "tiny_sd15"))
    if "unet_sdxl" in which:
        diag_unet(("sdxl",))
    if "unet_sd15" in which:
        diag_unet(("sd15",))
    if "bench_unet" in which:
        bench_unet()
    if "prof_unet" in which:
        prof_unet()
    if "prof_unet_sd15" in which:
        prof_unet("sd15", 4, 64)
    nbad = sum(1 for _, ok in RESULTS if not ok)
    print(f"=== {len(RESULTS) - nbad}/{len(RESULTS)} cases OK in {time.time() - t0:.1f}s ===", flush=True)
