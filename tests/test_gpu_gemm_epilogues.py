"""Kernel-level tests of the GEMM epilogue variants every transformer block runs, through the C ABI:
- the row-statistics producer (the GEMMs that write the residual stream also emit per-row partial sums Σx, Σx² of
  their fp16 output, one slot per column half of every N block), in every addend mode and in place;
- the LayerNorm-fold consumer, plain and GEGLU (`rstd·acc − rstd·mean·s_n + t_n` on the folded weight), with the
  statistics from torch or from a real producer run;
- the weight fold itself (`fp16(w·γ)`, s_n, t_n);
- the GEGLU activation over every finite fp16 gate value.
The statistics are checked against the fp64 sums of the kernel's own fp16 output within the worst-case bound of fp32
recursive summation, (n − 1)·2⁻²⁴·Σ|x| for n terms (taken as n·2⁻²⁴·Σ|x|). The fold replaces the reference's fp16
rounding of LayerNorm's output by the rounding of fp16(w·γ), so its error is judged against the exact (fp64)
LayerNorm → Linear on the same fp16 input, next to the error of the unfused op_layernorm → op_linear path. The plain
fp16 outputs (producer, in place, the chain's to_out, GEGLU) are gated element by element within the accumulation bound
of `test_gpu_gemm.py`."""
import numpy as np
import pytest
import torch

from test_gpu_gemm import check_bound, dev, linear_kblocks, rnd

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
ADD_MODES = ("none", "residual", "temb_staged", "temb_rows")
# the fold's cancellation (var = Σx²/C − mean², rstd·acc − rstd·mean·s_n, all fp32) grows with the rows' mean
# offset: at μ/σ ≤ 30 the fused error stays within 1.5x the unfused path's (observed 0.99-1.01x); beyond, envelopes
# ≈5x the largest observed error (H100 SXM 80GB, 400 W: 8.5e-4 at μ/σ = 100, 7.5e-3 at 300; DESIGN §3)
FOLD_ENVELOPE = {100: 4e-3, 300: 4e-2}
FOLD_FLOOR = 2e-5


@pytest.fixture(scope="module", autouse=True)
def _fp32_refs():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def addend_for(g, mode, M, N):
    """(addend, add_rows_per_group) of the four epilogue add modes: none, full residual, a time-embedding row per
    256 rows (every 128-row tile inside one sample: the row is staged in shared memory), a row per 48 rows (tiles
    span several samples: per-row global loads)."""
    if mode == "none":
        return None, 1
    if mode == "residual":
        return rnd(g, M, N), 1
    rpg = 256 if mode == "temb_staged" else 48
    return rnd(g, (M + rpg - 1) // rpg, N), rpg


def check_stats(out, stats, bn, what):
    """stats [2·ceil(N/bn), M, 2]: part p holds (Σx, Σx²) of out's columns [p·bn/2, (p+1)·bn/2) ∩ [0, N)."""
    M, N = out.shape
    half = bn // 2
    assert stats.shape == (2 * ((N + bn - 1) // bn), M, 2)
    assert torch.isfinite(stats).all(), f"{what}: a statistics slot was not written"
    o = out.double()
    worst = 0.0
    for p in range(stats.shape[0]):
        x = o[:, p * half:min((p + 1) * half, N)]
        for k, (exact, mag) in enumerate(((x.sum(1), x.abs().sum(1)), ((x * x).sum(1), (x * x).sum(1)))):
            err = (stats[p, :, k].double() - exact).abs()
            bound = half * U32 * mag
            assert bool((err <= bound).all()), \
                f"{what}: part {p} {'Σx' if k == 0 else 'Σx²'} off by {err.max().item():.3e} (bound {bound.max().item():.3e})"
            worst = max(worst, (err / bound.clamp_min(1e-300)).max().item())
    print(f"[epilogue] {what}: statistics within {worst:.3f} of the fp32 summation bound")


def pack_geglu(w, b):
    """GEGLU weight packing of the kernel: per 256-row tile, 128 value rows then the 128 matching gate rows."""
    inner = w.shape[0] // 2
    idx = []
    for t in range(inner // 128):
        idx += list(range(t * 128, t * 128 + 128)) + list(range(inner + t * 128, inner + t * 128 + 128))
    idx = torch.tensor(idx, device=w.device)
    return w[idx].contiguous(), (b[idx].contiguous() if b is not None else None)


def ln_exact(h, gamma, beta, eps=1e-5):
    x = h.double()
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * gamma.double() + beta.double()


def lnlinear_exact(h, gamma, beta, w, b, geglu):
    """LayerNorm → Linear (→ GEGLU) in fp64 on the fp16 input, w / b unpacked."""
    pre = ln_exact(h, gamma, beta) @ w.double().t()
    if b is not None:
        pre = pre + b.double()
    if not geglu:
        return pre
    inner = w.shape[0] // 2
    return pre[:, :inner] * torch.nn.functional.gelu(pre[:, inner:])


def torch_stats(h, parts):
    """[parts, M, 2] fp32 row (Σx, Σx²) over equal column slices, summed in fp64."""
    x = h.double().reshape(h.shape[0], parts, -1)
    return torch.stack([x.sum(2), (x * x).sum(2)], 2).permute(1, 0, 2).float().contiguous()


def fold_vs_unfused(nv, h, stats, gamma, beta, w, b, geglu, what, ratio, force_bn=0, force_streamk=False):
    """Runs the fused consumer and the unfused op_layernorm → op_linear path on h; returns (fused out, fused error,
    unfused error) vs the exact reference, and gates fused ≤ 1.5x unfused + floor (ratio ≤ 30) or the envelope.
    `force_streamk` applies to the fused consumer only: the unfused path stays the plain tile walk it is judged by."""
    wk, bk = pack_geglu(w, b) if geglu else (w, b)
    wf, s, t = nv.op_fold_ln(wk, gamma, beta, bk)
    fused = nv.op_linear_lnfold(h, wf, s, t, stats, geglu=geglu, force_bn=force_bn, force_streamk=force_streamk)
    unfused = nv.op_linear(nv.op_layernorm(h, gamma, beta), wk, bk, geglu=geglu)
    ref = lnlinear_exact(h, gamma, beta, w, b, geglu)
    ef, eu = rel_l2_64(fused, ref), rel_l2_64(unfused, ref)
    lim = 1.5 * eu + FOLD_FLOOR if ratio <= 30 else FOLD_ENVELOPE[ratio]
    print(f"[epilogue] {what} μ/σ={ratio}: fused rel-L2 {ef:.3e}, unfused {eu:.3e} (gate {lim:.2e})")
    assert ef <= lim, f"{what} μ/σ={ratio}: fused rel-L2 {ef:.3e} > {lim:.2e} (unfused {eu:.3e})"
    return fused, ef, eu


def gate_linear(what, out, a, w, bias=None, addend=None, rpg=1, bn=0, geglu=False, force_streamk=False):
    """op_linear's output gated per element; the launch's schedule decides whether the stream-K term applies."""
    from cfgpp_b200 import _native as nv
    sched = nv.linear_schedule(a, w, bias, addend, rpg, geglu=geglu, force_bn=bn, force_streamk=force_streamk)
    check_bound(what, out, linear_kblocks(a), w, a.shape[0], bias, addend, rpg, sched, geglu)


def rel_l2_64(a, ref):
    a, ref = a.double(), ref.double()
    return ((a - ref).norm() / (ref.norm() + 1e-300)).item()


# ---- producer statistics ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("mode", ADD_MODES)
@pytest.mark.parametrize("M", [300, 77])
def test_rowstats_producer(M, mode, bn):
    """N = 640: a partial last N block at BN = 256 (its upper column half is all padding and must sum to 0); M = 300 a
    partial last M tile, M = 77 a single partial tile."""
    from cfgpp_b200 import _native as nv
    N, K = 640, 320
    g = torch.Generator().manual_seed(M + bn + ADD_MODES.index(mode))
    a, w, bias = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5), rnd(g, N)
    addend, rpg = addend_for(g, mode, M, N)
    out, stats = nv.op_linear_stats(a, w, bn, bias, addend, rpg)
    what = f"rowstats {M}x{N}x{K} BN{bn} {mode}"
    gate_linear(what, out, a, w, bias, addend, rpg, bn)
    check_stats(out, stats, bn, what)
    if mode == "none":  # the statistics variant writes what the plain epilogue writes
        assert torch.equal(out, nv.op_linear(a, w, bias, force_bn=bn))


@pytest.mark.parametrize("M,N,K,bn", [(1000, 1280, 640, 128), (4096, 640, 640, 160), (77, 320, 512, 64),
                                      (2048, 1280, 5120, 256)])
def test_rowstats_producer_in_place(M, N, K, bn):
    """attn1.to_out / attn2.to_out / ff.out run with out == addend (the residual stream): bit-identical to the
    out-of-place run, statistics included."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(M + N + K)
    a, w, bias, tok = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5), rnd(g, N), rnd(g, M, N, shift=0.5)
    tok0 = tok.clone()
    oop, oop_stats = nv.op_linear_stats(a, w, bn, bias, tok0)
    out, stats = nv.op_linear_stats(a, w, bn, bias, tok, out=tok)
    assert out.data_ptr() == tok.data_ptr()
    what = f"rowstats in place {M}x{N}x{K} BN{bn}"
    gate_linear(what, tok, a, w, bias, tok0, 1, bn)
    check_stats(tok, stats, bn, what)
    assert torch.equal(tok, oop) and torch.equal(stats, oop_stats)
    tok.copy_(tok0)
    assert torch.equal(nv.op_linear(a, w, bias, tok, force_bn=bn, out=tok), oop)


# ---- the weight fold ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,K,hb", [(1536, 320, False), (3072, 640, False), (4608, 1280, False), (10240, 1280, True),
                                    (2560, 320, True), (1001, 640, True)])
def test_fold_ln(N, K, hb):
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(N + K)
    w, gamma, beta = rnd(g, N, K, scale=K ** -0.5), rnd(g, K, scale=0.2, shift=1.0), rnd(g, K, scale=0.2)
    bias = rnd(g, N) if hb else None
    wf, s, t = nv.op_fold_ln(w, gamma, beta, bias)
    assert torch.equal(wf, (w.float() * gamma.float()).half()), "wf != fp16(w * gamma)"
    wfd = wf.double()
    es, bs = (s.double() - wfd.sum(1)).abs(), K * U32 * wfd.abs().sum(1)
    bw = beta.double() * w.double()
    tx = bw.sum(1) + (bias.double() if hb else 0.0)
    et, bt = (t.double() - tx).abs(), (K + 1) * U32 * (bw.abs().sum(1) + (bias.double().abs() if hb else 0.0))
    print(f"[epilogue] fold_ln {N}x{K}: s within {(es / bs).max().item():.3f}, t within {(et / bt).max().item():.3f} "
          f"of the fp32 summation bound")
    assert bool((es <= bs).all()) and bool((et <= bt).all())


# ---- the LayerNorm-fold consumer ------------------------------------------------------------------------------------
def padded_qkv_rows(C):
    """3·Cp of SD v1.5's self-attention: 8 heads of C / 8 columns, zero-padded to a multiple of 64 per head."""
    hd = C // 8
    return 3 * 8 * ((hd + 63) // 64 * 64)


def consumer_cases():
    for C in (320, 640, 1280):
        for src in ["torch"] + [bn for bn in (64, 128, 160, 256) if C % bn == 0]:
            for geglu in (False, True):
                yield C, src, geglu


@pytest.mark.parametrize("C,src,geglu", list(consumer_cases()))
def test_lnfold_consumer(C, src, geglu):
    """Statistics from torch (the consumer alone, C / 32 parts) or from a producer run at tile width src (the
    residual add of attn / ff output, 2·C/BN parts); rows offset by μ/σ ∈ {0, 3, 30, 100, 300}."""
    from cfgpp_b200 import _native as nv
    M = 1000
    N = 8 * C if geglu else padded_qkv_rows(C)
    g = torch.Generator().manual_seed(C + N + (0 if src == "torch" else src))
    gamma, beta = rnd(g, C, scale=0.2, shift=1.0), rnd(g, C, scale=0.2)
    w, b = rnd(g, N, C, scale=C ** -0.5), rnd(g, N)
    for ratio in (0, 3, 30, 100, 300):
        if src == "torch":
            h = rnd(g, M, C, shift=float(ratio))
            stats = torch_stats(h, C // 32)
        else:
            Kp = 512
            a, wp, bp = rnd(g, M, Kp), rnd(g, C, Kp, scale=Kp ** -0.5 * 0.8), rnd(g, C, scale=0.2)
            h, stats = nv.op_linear_stats(a, wp, src, bp, rnd(g, M, C, scale=0.6, shift=float(ratio)))
            check_stats(h, stats, src, f"producer {M}x{C} BN{src}")
        fold_vs_unfused(nv, h, stats, gamma, beta, w, b if geglu else None, geglu,
                        f"lnfold{' geglu' if geglu else ''} {M}x{N}x{C} stats:{src}", ratio)


def test_lnfold_consumer_rejects_bias():
    """The fold consumer's bias lives in t_n; a bias vector next to the statistics would be ignored, so it is refused."""
    import ctypes
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(3)
    h, w, bias = rnd(g, 128, 64), rnd(g, 64, 64), rnd(g, 64)
    wf, s, t = nv.op_fold_ln(w, rnd(g, 64), rnd(g, 64))
    stats = torch_stats(h, 2)
    out = torch.empty(128, 64, dtype=torch.float16, device=dev)
    lib = nv.load()
    st = lib.cfgpp_op_linear_lnfold(nv.ptr(h), nv.ptr(wf), 128, 64, 64, nv.ptr(bias), None, 0, 1, nv.ptr(out), 64, 0, 0,
                                    0, None, nv.ptr(stats), 2, ctypes.c_float(1e-5), nv.ptr(s), nv.ptr(t), nv.stream_ptr())
    assert st != 0 and b"bias" in lib.cfgpp_last_error()


def producer_bn(nv, attn, wo, bo, tok):
    """The tile width the UNet's LayerNorm-fold producer takes (`producer` in unet.cu): the launch's own schedule, or
    when that width does not divide C the first of 160, 128, 64 that does."""
    C = wo.shape[0]
    bn = nv.linear_schedule(attn, wo, bo, tok, out=tok)["bn"]
    return bn if C % bn == 0 else next(b for b in (160, 128, 64) if C % b == 0)


UNET_CHAINS = [  # (M, C) at UNet batch 4 on the production latents: every transformer level
    pytest.param(4 * 64 * 64, 768, id="sdxl_refiner-1024x1024-C768"),
    pytest.param(4 * 32 * 32, 1536, id="sdxl_refiner-1024x1024-C1536"),
    pytest.param(4 * 16 * 16, 1536, id="sdxl_refiner-1024x1024-mid-C1536"),
    pytest.param(4 * 76 * 52, 768, id="sdxl_refiner-832x1216-C768"),
    pytest.param(4 * 38 * 26, 1536, id="sdxl_refiner-832x1216-C1536"),
    pytest.param(4 * 96 * 96, 320, id="sd2-768x768-C320"),
    pytest.param(4 * 48 * 48, 640, id="sd2-768x768-C640"),
    pytest.param(4 * 24 * 24, 1280, id="sd2-768x768-C1280"),
    pytest.param(4 * 12 * 12, 1280, id="sd2-768x768-mid-C1280"),
]


@pytest.mark.parametrize("M,C", UNET_CHAINS)
def test_lnfold_chain_production(M, C):
    """The chain of `test_lnfold_chain_as_unet` at the SDXL refiner's and SD 2's widths and production M (head dim 64:
    Cp = C), with the producer at the tile width the UNet picks, so the consumers see the real count of partial
    statistics (2·C / BN: up to 24 at C = 1536)."""
    lnfold_chain(M, C, C, None, seed=M + C + 1, reps=3)


@pytest.mark.parametrize("M,C,Cp,bn", [(16384, 640, 640, 128), (4096, 1280, 1280, 256), (8192, 320, 512, 160),
                                       (2048, 1280, 1536, 64)])
def test_lnfold_chain_as_unet(M, C, Cp, bn):
    """The transformer block's wiring: to_out writes `tok` in place (+ residual) and its statistics, then
    to_qkv(+norm1) and ff.geglu(+norm3) read `tok` with the same statistics buffer. SDXL (C = 640 / 1280, head dim 64)
    and SD v1.5 (padded heads Cp) shapes. Twelve repetitions are bit-identical."""
    lnfold_chain(M, C, Cp, bn, seed=M + C, reps=12)


def lnfold_chain(M, C, Cp, bn, seed, reps):
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(seed)
    attn, wo, bo = rnd(g, M, Cp), rnd(g, C, Cp, scale=Cp ** -0.5), rnd(g, C)
    tok0 = rnd(g, M, C, shift=0.5)
    gamma, beta = rnd(g, C, scale=0.2, shift=1.0), rnd(g, C, scale=0.2)
    wqkv = rnd(g, 3 * Cp, C, scale=C ** -0.5)
    wff, bff = rnd(g, 8 * C, C, scale=C ** -0.5), rnd(g, 8 * C)
    wffp, bffp = pack_geglu(wff, bff)
    fq = nv.op_fold_ln(wqkv, gamma, beta)
    ff = nv.op_fold_ln(wffp, gamma, beta, bffp)
    tok = tok0.clone()

    def run():
        tok.copy_(tok0)
        _, stats = nv.op_linear_stats(attn, wo, bn, bo, tok, out=tok)
        qkv = nv.op_linear_lnfold(tok, *fq, stats)
        hff = nv.op_linear_lnfold(tok, *ff, stats, geglu=True)
        return tok.clone(), stats, qkv, hff

    if bn is None:
        bn = producer_bn(nv, attn, wo, bo, tok)
    first = run()
    what = f"chain {M}x{C} Cp{Cp} BN{bn} ({2 * -(-C // bn)} statistics parts)"
    gate_linear(what + " to_out", first[0], attn, wo, bo, tok0, 1, bn)
    check_stats(first[0], first[1], bn, what)
    for name, got, w, b, geglu in (("to_qkv", first[2], wqkv, None, False), ("ff.geglu", first[3], wff, bff, True)):
        ref = lnlinear_exact(first[0], gamma, beta, w, b, geglu)
        unfused = nv.op_linear(nv.op_layernorm(first[0], gamma, beta), *(pack_geglu(w, b) if geglu else (w, b)),
                               geglu=geglu)
        ef, eu = rel_l2_64(got, ref), rel_l2_64(unfused, ref)
        print(f"[epilogue] {what} {name}(+norm): fused rel-L2 {ef:.3e}, unfused {eu:.3e}")
        assert ef <= 1.5 * eu + FOLD_FLOOR
    for _ in range(reps):
        again = run()
        assert all(torch.equal(x, y) for x, y in zip(again, first))


# ---- GEGLU --------------------------------------------------------------------------------------------------------
def fp16_ulp_key(x):
    """fp16 values as ordered integers (±0 → 0): the difference of two keys is their distance in ulps."""
    b = x.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    return torch.where(b >= 0x8000, 0x8000 - b, b)


def test_geglu_every_finite_fp16_gate():
    """One-hot A rows (K = 64) and all-ones value rows make acc equal the packed weights, so the 1024 gate rows carry
    all 63,488 finite fp16 values through the real epilogue: fp16(gelu) within 1 ulp of fp16(exact erf-GELU)."""
    from cfgpp_b200 import _native as nv
    bits = np.arange(65536, dtype=np.uint32).astype(np.uint16).view(np.float16)
    vals = bits[np.isfinite(bits)]
    assert vals.size == 63488
    gates = np.zeros(1024 * 64, dtype=np.float16)
    gates[:vals.size] = vals
    G = torch.from_numpy(gates.reshape(1024, 64)).to(dev)  # gate row j, one-hot position k
    w = torch.ones(2048, 64, dtype=torch.float16, device=dev)
    for t in range(8):
        w[256 * t + 128:256 * t + 256] = G[128 * t:128 * t + 128]
    a = torch.eye(64, dtype=torch.float16, device=dev)
    got = nv.op_linear(a, w, geglu=True).t()  # [1024, 64]: got[j, k] = GEGLU of gate value G[j, k]
    ref = torch.nn.functional.gelu(G.double()).half()
    d = (fp16_ulp_key(got) - fp16_ulp_key(ref)).abs()
    n1 = int((d.reshape(-1)[:vals.size] == 1).sum())
    print(f"[epilogue] geglu over {vals.size} finite fp16 gates: max {int(d.max())} ulp, {n1} at 1 ulp")
    assert int(d.max()) <= 1, f"worst gate {G.reshape(-1)[d.reshape(-1).argmax()].item()}: {int(d.max())} ulp"


@pytest.mark.parametrize("C", [320, 640, 1280])
@pytest.mark.parametrize("M", [77, 1000])
@pytest.mark.parametrize("hb", [True, False])
def test_geglu_shapes(C, M, hb):
    """ff.net.0 at N = 8C for every channel count of the UNets, ragged M, with and without bias."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(C + M + hb)
    inner = 4 * C
    a, w = rnd(g, M, C), rnd(g, 2 * inner, C, scale=C ** -0.5)
    b = rnd(g, 2 * inner) if hb else None
    wp, bp = pack_geglu(w, b)
    out = nv.op_linear(a, wp, bp, geglu=True)
    gate_linear(f"geglu {M}x{inner}x{C}{' +bias' if hb else ''}", out, a, wp, bp, geglu=True)


# ---- stream-K -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("force_streamk", [False, True])
@pytest.mark.parametrize("kind", ["rowstats", "lnfold", "geglu", "lnfold_geglu"])
def test_epilogue_streamk_repeatable(kind, force_streamk):
    """Shapes with a remainder of tiles over the 132 SMs (rowstats 32x10 tiles, lnfold 32x15, GEGLU 32x20), so with the
    stream-K split forced on the fix-up path feeds each epilogue: result gated, 12 launches bit-identical."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(len(kind))
    M = 4096
    if kind == "rowstats":
        N, K, bn = 1280, 1280, 128
        a, w, bias, res = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5), rnd(g, N), rnd(g, M, N)
        run = lambda: nv.op_linear_stats(a, w, bn, bias, res, force_streamk=force_streamk)
        first = run()
        gate_linear(f"rowstats(stream-K) {M}x{N}x{K}", first[0], a, w, bias, res, 1, bn, force_streamk=force_streamk)
        check_stats(first[0], first[1], bn, f"rowstats(stream-K) {M}x{N}x{K}")
    elif kind == "geglu":
        C = 640
        a, w, b = rnd(g, M, C), rnd(g, 8 * C, C, scale=C ** -0.5), rnd(g, 8 * C)
        wp, bp = pack_geglu(w, b)
        run = lambda: (nv.op_linear(a, wp, bp, geglu=True, force_streamk=force_streamk),)
        first = run()
        gate_linear(f"geglu(stream-K) {M}x{4 * C}x{C}", first[0], a, wp, bp, geglu=True, force_streamk=force_streamk)
    else:
        geglu = kind == "lnfold_geglu"
        C = 640 if geglu else 1280
        N = 8 * C if geglu else 3 * C
        h = rnd(g, M, C, shift=1.0)
        gamma, beta = rnd(g, C, scale=0.2, shift=1.0), rnd(g, C, scale=0.2)
        w, b = rnd(g, N, C, scale=C ** -0.5), rnd(g, N)
        stats = torch_stats(h, C // 32)
        fused, _, _ = fold_vs_unfused(nv, h, stats, gamma, beta, w, b, geglu, f"lnfold(stream-K) {M}x{N}x{C}", 1,
                                      force_streamk=force_streamk)
        wk, bk = pack_geglu(w, b) if geglu else (w, b)
        wf, s, t = nv.op_fold_ln(wk, gamma, beta, bk)
        run = lambda: (nv.op_linear_lnfold(h, wf, s, t, stats, geglu=geglu, force_streamk=force_streamk),)
        first = run()
        assert torch.equal(first[0], fused)
    for _ in range(12):
        assert all(torch.equal(x, y) for x, y in zip(run(), first))
