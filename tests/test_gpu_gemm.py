"""Kernel-level tests of the wgmma GEMM / implicit-GEMM 3x3 convolution (`gemm_kernel` in `gemm.cu`), element by
element, through `op_linear`, `op_linear_stats` and `op_conv3x3_ex`.

Every launch's schedule (tile width BN, grid, stream-K split and its pieces per tile, A-tile mode) is read back with
`linear_schedule` / `conv3x3_schedule` (the debug entry point `cfgpp_dbg_gemm_schedule`), which build the op exactly as
the launch does. A test that names a path asserts it takes it, and the last test of the module asserts that every tile
width, both convolution A-tile modes, natural and forced stream-K, a tile split over three or more pieces and every
addend mode ran under the per-element gates. The schedule depends on the card's SM count, so nothing here guesses it.

Family A, integer known answers (bit-exact). A and W are small integers (A in [-2, 2], W sparse in {±1, ±2}, at most
511 non-zeros per row, so every |exact| < 2048, which is asserted); bias, residual and time-embedding rows are integers.
Every product and partial sum is then an integer below 2^24, exact in fp32 whatever the summation order, the stream-K
split or the accumulator's rounding mode, so the output must be bit-identical to fp16(exact), or with an addend to
fp16(fp16(exact + bias) + addend), at every element. Variants: W times 2^-24 (outputs in fp16's subnormal range), a bias
that puts the outputs across ±65504 (overflow to ±inf exactly as `.half()` does), and GEGLU with every gate
pre-activation an integer >= 8, for which fp16(gelu(g)) = g; `assert_gelu_identity` checks that through the kernel's own
GELU for every gate value used, so the value / gate pairing of the 256-row packing is pinned bit-exactly.

Family B, float inputs under a per-element bound. The reference is fp64 on the GPU from the same fp16 operands, in the
kernel's k order (a convolution's k = tap·Cin + c: nine shifted row gathers of the zero-padded NHWC input, not conv2d).
With p_k = a_{m,k}·w_{n,k} (exact in fp64), P_b the prefix sum over the first 64·b products (the k-blocks of the main
loop), ε = 2^-23 and u = 2^-24:
  E_acc = 2ε·(4·Σ_b |P_b| + 5·Σ_k |p_k|)                (+ ε·(K/16 + 3)·max_j |S_j|  when the launch takes stream-K)
  E_t   = E_acc + u·|ref_t| + ½·ulp16(|ref_t| + E_acc),    ref_t = P_{K/64} + bias
  E     = E_t + u·|ref| + ½·ulp16(|ref| + E_t),           ref = ref_t + addend     (with an addend)
E_acc charges two truncated fp32 units (2ε) per wgmma k16 step on the running sum S_{j-1} and on the step's operand
magnitudes, 2ε·(Σ_{j=1}^{K/16} |S_{j-1}| + Σ_k |p_k|): one for aligning the step's products to the largest exponent, one
for normalising the sum, both truncated. PTX documents only "fp32 accumulation", and published studies of earlier tensor
cores found truncation at both points, so round-to-nearest is not assumed. (A single unit per step is not enough on an
H100: the bias-cancellation family reached 1.26x such a bound in a one-tile launch without stream-K, where the kernel
does nothing but issue the k16 steps in order and add the bias.) The k16 prefixes
inside k-block b are bounded by |P_b| + Σ_{k in b} |p_k|, four steps per block, which gives the per-k-block form above.
The stream-K term covers pieces that restart from zero (their running sums differ from S_j by at most max_j |S_j|,
bounded per block the same way) and the <= 3 fp32 adds of parked partials. u·|ref_t| is the bias add, ½ ulp16 the
rounding to fp16 (the same two for the addend). GEGLU carries the value's and the gate's E_t through
fp16(fp16(a)·fp16(gelu(fp16(g)))): gelu is 1.13-Lipschitz and the kernel's fp16(gelu) lies within 1 ulp of
fp16(exact) over every fp16 gate (`test_geglu_every_finite_fp16_gate`), so
  E_ge = 1.13·E_g + 2.5·ulp16(|G| + 1.13·E_g),   E = E_a·(|G| + E_ge) + |a|·E_ge + u·(|a| + E_a)·(|G| + E_ge) (+ ½ ulp16).
Input families: flat (randn, W·K^-½), cancellation (rows of A at mean 100σ against zero-sum weight rows: small outputs,
large partials), all-positive (|A|, |W|: the worst case for a truncating accumulator; its mean signed error is printed),
dynamic range (row scales 2^-8..2^8, column scales 2^-8..2^0), bias cancellation (a bias that cancels a large
accumulator) and softmax rows (non-negative fp16 rows summing to 1, flat and peaked, against V at mean 10σ: the VAE's
P·V at K = 16384). Every case asserts a finite output (except the overflow cases) and prints max |err|/E and rel-L2.

The production launches are derived from the model configs at the sizes of `production.py` (every full-size UNet at
each of its latent sizes, UNet batch 4; the VAE decoder and encoder at each image size; every text tower at
M = B·77; the ControlNets, vision towers, IP-Adapters and T2I-Adapters), run once per distinct launch signature in
their production layouts; `test_unet_launch_list_matches_profile` checks the derived UNet GEMM and attention lists
against the launches the native UNet reports, `test_t2i_adapter_launch_list_matches_plan_flops` the T2I-Adapter's
against its plan's FLOPs. The LayerNorm-fold consumers run their shapes as plain linears here (the fold arithmetic has
its own relative gate in `test_gpu_gemm_epilogues.py`)."""
import zlib

import pytest
import torch
import torch.nn.functional as F

import production as P
from test_gpu_norms import Gate, ulp16

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
EPS = 2.0 ** -23
U = 2.0 ** -24
PIECE = 1 << 24  # fp64 elements of one [rows, N] slice of the reference
SEEN = {"bn": set(), "a_mode": set(), "streamk": set(), "pieces3": 0, "addend": set(), "cases": 0, "forced": 0,
        "t2i_conv": set()}


@pytest.fixture(scope="module", autouse=True)
def _fp64_refs():
    torch.backends.cuda.matmul.allow_tf32 = False


def rnd(g, *s, scale=1.0, shift=0.0):
    """fp16 N(shift, scale²) from a CPU generator (seeded shapes do not depend on the device's RNG)."""
    return (torch.randn(*s, generator=g) * scale + shift).half().to(dev)


def gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


# ------------------------------------------------------------------------------------------------ schedules

def record(sched, modes, *, streamk=None, pieces3=False, forced=False):
    """Note what a gated launch covered (`forced`: its tile width, stream-K split or A tile was forced); assert the
    path its test names."""
    if streamk is not None:
        assert sched["streamk"] == streamk, f"expected stream-K {streamk}, schedule {sched}"
    if pieces3:
        assert sched["max_pieces"] >= 3, f"expected tiles of >= 3 pieces, schedule {sched}"
    SEEN["bn"].add(sched["bn"])
    SEEN["a_mode"].add(sched["a_mode"])
    SEEN["streamk"].add(sched.get("sk_kind") if sched["streamk"] else None)
    SEEN["pieces3"] += sched["max_pieces"] >= 3
    SEEN["addend"] |= modes
    SEEN["cases"] += 1
    SEEN["forced"] += forced


def addend_modes(addend, rpg, M):
    """The epilogue's addend paths a launch takes: a time-embedding row is staged in shared memory for the 128-row tiles
    inside one sample, and loaded per row for the tiles that span samples."""
    if addend is None:
        return {"none"}
    if rpg <= 1:
        return {"residual"}
    return {"temb_staged" if m0 // rpg == min(m0 + 127, M - 1) // rpg else "temb_rows" for m0 in range(0, M, 128)}


# ------------------------------------------------------------------------------------------------ operands in k order

def linear_kblocks(a, a2=None):
    """fp64 k-blocks [rows, 64] of rows [r0, r1) of cat([a, a2], 1), in the kernel's k order."""
    def blocks(r0, r1):
        for src in (a, a2):
            if src is not None:
                x = src[r0:r1]
                for k in range(0, x.shape[1], 64):
                    yield x[:, k:k + 64].double()
    return blocks


def conv_kblocks(x, stride, pad):
    """fp64 k-blocks of the implicit GEMM of a 3x3 convolution on NHWC x: tap-major (k = tap·Cin + c), output pixel
    (y, x) of tap (kh, kw) reading input (stride·y + kh − pad, stride·x + kw − pad), zero outside the image."""
    B, H, W, Cin = x.shape
    Ho, Wo = H // stride, W // stride
    xp = F.pad(x, (0, 0, pad, 1, pad, 1))

    def blocks(r0, r1):
        r = torch.arange(r0, r1, device=dev)
        b, rem = r // (Ho * Wo), r % (Ho * Wo)
        y, xx = rem // Wo, rem % Wo
        for tap in range(9):
            kh, kw = divmod(tap, 3)
            at = xp[b, y * stride + kh, xx * stride + kw]
            for c in range(0, Cin, 64):
                yield at[:, c:c + 64].double()
    return blocks


def slices(blocks, w, M, bounds, streamk=False):
    """(r0, r1, S, E_acc) over row slices: S = the fp64 product, E_acc the accumulation bound (None if not bounds)."""
    N, K = w.shape
    w64 = w.double()
    wabs = w64.abs() if bounds else None
    rows = max(1, PIECE // N)
    for r0 in range(0, M, rows):
        r1 = min(M, r0 + rows)
        S = torch.zeros(r1 - r0, N, dtype=torch.float64, device=dev)
        if bounds:
            sum_p, sum_abs = torch.zeros_like(S), torch.zeros_like(S)
            max_s = torch.zeros_like(S) if streamk else None
        for kb, ab in enumerate(blocks(r0, r1)):
            wb = w64[:, kb * 64:(kb + 1) * 64]
            if bounds:
                sum_p += S.abs()
                blk_abs = ab.abs() @ wabs[:, kb * 64:(kb + 1) * 64].t()
                sum_abs += blk_abs
                if streamk:
                    torch.maximum(max_s, S.abs() + blk_abs, out=max_s)
            S += ab @ wb.t()
        assert (kb + 1) * 64 == K, "k-blocks do not cover K"
        e = None
        if bounds:
            e = 2 * EPS * (4 * sum_p + 5 * sum_abs)
            if streamk:
                e += EPS * (K / 16 + 3) * max_s
            del sum_p, sum_abs, max_s
        yield r0, r1, S, e


def addend_rows(addend, rpg, r0, r1):
    if rpg <= 1:
        return addend[r0:r1]
    return addend[torch.arange(r0, r1, device=dev) // rpg]


def geglu_cols(N):
    """Packed GEGLU columns: output j takes value row 256·(j / 128) + j % 128 and the gate row 128 below it."""
    j = torch.arange(N // 2, device=dev)
    v = (j // 128) * 256 + j % 128
    return v, v + 128


# ------------------------------------------------------------------------------------------------ the two gates

def check_bound(what, out, blocks, w, M, bias=None, addend=None, rpg=1, sched=None, geglu=False, signed=False,
                scale=None):
    """Family B: every element of out [M, n_out] within E of fp64 (module docstring). Returns the worst |err|/E. With
    `scale` s (the scaled-residual epilogue, fp16(addend + fp16(fp16(t)·s))) the addend terms follow
      E_s = |s|·E_t + u·|s·ref_t| + ½·ulp16(|s·ref_t| + |s|·E_t),   ref = s·ref_t + addend."""
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    sk = bool(sched and sched["streamk"])
    gate = Gate(what)
    sdiff = torch.zeros((), dtype=torch.float64, device=dev)
    for r0, r1, S, e_acc in slices(blocks, w, M, True, sk):
        pre = S + bias.double() if bias is not None else S
        e_t = e_acc + U * pre.abs()
        o = out[r0:r1].double()
        if geglu:
            vi, gi = geglu_cols(w.shape[0])
            e_t = e_t + 0.5 * ulp16(pre.abs() + e_t)
            a, ea, g, eg = pre[:, vi], e_t[:, vi], pre[:, gi], e_t[:, gi]
            G = F.gelu(g)
            e_ge = 1.13 * eg + 2.5 * ulp16(G.abs() + 1.13 * eg)
            ref = a * G
            bound = ea * (G.abs() + e_ge) + a.abs() * e_ge + U * (a.abs() + ea) * (G.abs() + e_ge)
        elif addend is not None:
            e_t = e_t + 0.5 * ulp16(pre.abs() + e_t)
            if scale is not None:
                pre = scale * pre
                e_t = abs(scale) * e_t + U * pre.abs() + 0.5 * ulp16(pre.abs() + abs(scale) * e_t)
            ref = pre + addend_rows(addend, rpg, r0, r1).double()
            bound = e_t + U * ref.abs()
        else:
            ref, bound = pre, e_t
        gate.add(o, ref, bound)
        if signed:
            sdiff += ((o.abs() - ref.abs()) / (bound + 0.5 * ulp16(ref.abs() + bound))).sum()
    worst = gate.done("gemm")
    if signed:
        print(f"[gemm] {what}: mean signed (|out| - |ref|)/E {sdiff.item() / out.numel():+.4f}")
    return worst


def check_exact(what, out, blocks, w, M, bias=None, addend=None, rpg=1, geglu=False, limit=2048.0, finite=True,
                scale=None):
    """Family A: out [M, n_out] bit-identical to the fp16 rounding chain of the exact (fp64) integer result (with
    `scale` s: fp16(addend + fp16(fp32(fp16(exact + bias))·s)))."""
    if finite:
        assert torch.isfinite(out).all(), f"{what}: non-finite output"
    bad, mx = 0, 0.0
    for r0, r1, S, _ in slices(blocks, w, M, False):
        mx = max(mx, S.abs().max().item())
        t = (S + bias.double() if bias is not None else S).float().half()
        if geglu:
            vi, gi = geglu_cols(w.shape[0])
            t = (t[:, vi].float() * t[:, gi].float()).half()
        elif addend is not None:
            if scale is not None:
                t = (t.float() * torch.tensor(scale, dtype=torch.float32, device=dev)).half()
            t = (t.float() + addend_rows(addend, rpg, r0, r1).float()).half()
        o = out[r0:r1]
        neq = ~((o == t) | (torch.isnan(o) & torch.isnan(t)))
        if neq.any():
            bad += int(neq.sum())
            r, c = neq.nonzero()[0].tolist()
            first = (r0 + r, c, o[r, c].item(), t[r, c].item())
    assert mx < limit, f"{what}: exact result {mx} reaches the operand bound {limit}"
    print(f"[gemm exact] {what}: {'bit-exact' if not bad else f'{bad} elements differ'} (max |exact| {mx:g})")
    assert not bad, f"{what}: {bad} elements differ from fp16(exact); first (row, col, got, want) = {first}"


# ------------------------------------------------------------------------------------------------ operand families

def int_act(g, *s):
    return torch.randint(-2, 3, s, generator=g, device=dev).half()


def int_weight(g, N, K, nnz=511):
    """Integer rows with min(K, nnz) non-zeros in {±1, ±2}: against A in [-2, 2], |exact| <= 4·nnz < 2048."""
    nnz = min(K, nnz)
    idx = torch.rand(N, K, generator=g, device=dev).argsort(1)[:, :nnz]
    val = torch.randint(1, 3, (N, nnz), generator=g, device=dev) * (torch.randint(0, 2, (N, nnz), generator=g,
                                                                                   device=dev) * 2 - 1)
    return torch.zeros(N, K, device=dev).scatter_(1, idx, val.float()).half()


def int_vec(g, *s, lo=-16, hi=16):
    return torch.randint(lo, hi + 1, s, generator=g, device=dev).half()


FAMILIES = ("flat", "cancellation", "all_positive", "dynamic_range", "bias_cancel")


def float_operands(family, g, M, N, K):
    """(a [M, K], w [N, K], bias [N] or None) fp16 of one Family-B input family."""
    a = torch.randn(M, K, generator=g, device=dev)
    w = torch.randn(N, K, generator=g, device=dev) * K ** -0.5
    bias = torch.randn(N, generator=g, device=dev)
    if family == "cancellation":  # rows of A at mean 100σ, weight rows of zero sum
        a = a + 100.0
        w = w - w.mean(1, keepdim=True)
    elif family == "all_positive":
        a, w, bias = a.abs(), w.abs(), bias.abs()
    elif family == "dynamic_range":
        a = a * torch.exp2(torch.randint(-8, 9, (M, 1), generator=g, device=dev).float())
        w = w * torch.exp2(torch.randint(-8, 1, (N, 1), generator=g, device=dev).float())
    elif family == "bias_cancel":  # |acc| ≈ 100·sqrt(K)·|mean w|, cancelled by the bias down to O(1)
        a = a + 100.0
        w = w + torch.randn(N, 1, generator=g, device=dev) * K ** -0.5
        bias = None
    a, w = a.half(), w.half()
    if family == "bias_cancel":
        bias = -(100.0 * w.double().sum(1)).half()
    return a, w, (bias.half() if bias is not None else None)


def softmax_rows(g, M, K, peaked):
    s = torch.randn(M, K, generator=g, device=dev) * (8.0 if peaked else 1.0)
    return torch.softmax(s, 1).half()


# ------------------------------------------------------------------------------------------------ one launch, both gates

def run_linear(what, a, w, *, bias=None, addend=None, rpg=1, a2=None, geglu=False, force_bn=0, force_streamk=False,
               in_place=False, family=None, expect_sk=None, pieces3=False, signed=False):
    """Launch op_linear, read its schedule, gate it (family None: Family A bit-exact, else Family B)."""
    from cfgpp_b200 import _native as nv
    M = a.shape[0]
    kw = dict(bias=bias, add_rows_per_group=rpg, a2=a2, geglu=geglu, force_bn=force_bn, force_streamk=force_streamk)
    add0 = addend.clone() if (in_place and addend is not None) else addend
    sched = nv.linear_schedule(a, w, addend=addend, **kw)
    if force_streamk and sched["streamk"]:
        sched["sk_kind"] = "forced"
    elif sched["streamk"]:
        sched["sk_kind"] = "natural"
    out = nv.op_linear(a, w, addend=addend, out=addend if in_place else None, **kw)
    modes = addend_modes(addend, rpg, M)
    record(sched, modes, streamk=expect_sk, pieces3=pieces3, forced=bool(force_bn or force_streamk))
    mode = "+".join(sorted(modes)) + (" in place" if in_place else "")
    tag = (f"{what} BN{sched['bn']} grid {sched['grid']} tiles {sched['tiles']}"
           f"{' stream-K x' + str(sched['max_pieces']) if sched['streamk'] else ''} {mode}")
    blocks = linear_kblocks(a, a2)
    if family is None:
        check_exact(tag, out, blocks, w, M, bias, add0, rpg, geglu)
    else:
        check_bound(f"{tag} [{family}]", out, blocks, w, M, bias, add0, rpg, sched, geglu, signed)
    return out, sched


def run_conv(what, x, w, *, bias=None, addend=None, rpg=1, stride=1, pad=1, force_im2col=False, force_bn=0,
             family=None, expect_sk=None, expect_mode=None, pieces3=False, limit=2048.0, finite=True):
    from cfgpp_b200 import _native as nv
    B, H, W, Cin = x.shape
    M = B * (H // stride) * (W // stride)
    kw = dict(bias=bias, add_rows_per_group=rpg, stride=stride, pad=pad, force_im2col=force_im2col, force_bn=force_bn)
    sched = nv.conv3x3_schedule(x, w, addend=addend, **kw)
    if sched["streamk"]:
        sched["sk_kind"] = "natural"
    if expect_mode is not None:
        assert sched["a_mode"] == expect_mode, f"{what}: expected the {expect_mode} A tile, schedule {sched}"
    out = nv.op_conv3x3_ex(x, w, addend=addend, **kw).reshape(M, w.shape[0])
    modes = addend_modes(addend, rpg, M)
    record(sched, modes, streamk=expect_sk, pieces3=pieces3, forced=bool(force_bn or force_im2col))
    mode = "+".join(sorted(modes))
    tag = (f"{what} s{stride}p{pad} {sched['a_mode']} BN{sched['bn']} tiles {sched['tiles']}"
           f"{' stream-K x' + str(sched['max_pieces']) if sched['streamk'] else ''} {mode}")
    blocks = conv_kblocks(x, stride, pad)
    if family is None:
        check_exact(tag, out, blocks, w, M, bias, addend, rpg, limit=limit, finite=finite)
    else:
        check_bound(f"{tag} [{family}]", out, blocks, w, M, bias, addend, rpg, sched)
    return out, sched


def run_scaled_residual(what, a, w, bias, addend, s, family=None):
    """Launch op_linear_scaled_residual in place into `addend` with s an fp32 device word, read its schedule, gate it."""
    from cfgpp_b200 import _native as nv
    M = a.shape[0]
    s32 = torch.tensor([s], dtype=torch.float32, device=dev)
    add0 = addend.clone()
    sched = nv.linear_schedule(a, w, bias, addend)
    nv.op_linear_scaled_residual(a, w, addend, s32, bias, out=addend)
    record(sched, {"scaled_residual"})
    tag = f"{what} s {s} BN{sched['bn']} grid {sched['grid']} tiles {sched['tiles']} scaled_residual in place"
    if family is None:
        check_exact(tag, addend, linear_kblocks(a), w, M, bias, add0, scale=s32.item())
    else:
        check_bound(f"{tag} [{family}]", addend, linear_kblocks(a), w, M, bias, add0, sched=sched, scale=s32.item())
    return addend


def assert_gelu_identity(values):
    """fp16(gelu(g)) == g through the kernel's own GELU for every fp16 value g given (one-hot A, all-ones value rows)."""
    from cfgpp_b200 import _native as nv
    vals = torch.unique(values.reshape(-1).half())
    n = vals.numel()
    rows = -(-n // 64)
    G = torch.zeros(-(-rows // 128) * 128 * 64, dtype=torch.float16, device=dev)
    G[:n] = vals
    G = G.reshape(-1, 64)
    w = torch.ones(2 * G.shape[0], 64, dtype=torch.float16, device=dev)
    for t in range(G.shape[0] // 128):
        w[256 * t + 128:256 * t + 256] = G[128 * t:128 * t + 128]
    got = nv.op_linear(torch.eye(64, dtype=torch.float16, device=dev), w, geglu=True).t().reshape(-1)[:n]
    assert torch.equal(got, vals), f"fp16(gelu(g)) != g for g = {vals[got != vals][:8].tolist()}"


# ================================================================================================= edge sweep: linear

M_SWEEP = (1, 77, 127, 128, 129, 255, 257, 1000, 3952)
N_SWEEP = (8, 56, 64, 72, 160, 200, 264, 1000)
K_CYCLE = (64, 128, 320, 640, 1280, 2048)


def bns_for(N):
    return [0] + [bn for bn in (64, 128, 160, 256) if bn != 160 or N % 160 == 0]


@pytest.mark.parametrize("M", M_SWEEP)
def test_linear_edges_exact(M):
    """Family A over every N of the sweep at every forced tile width (and the default), K cycling 64..2048, bias and
    the addend modes rotating."""
    g = gen(M)
    for i, N in enumerate(N_SWEEP):
        K = K_CYCLE[(i + M) % len(K_CYCLE)]
        a, w, bias = int_act(g, M, K), int_weight(g, N, K), int_vec(g, N)
        for j, bn in enumerate(bns_for(N)):
            kind = (i + j) % 3
            addend, rpg = None, 1
            if kind == 1:
                addend = int_vec(g, M, N)
            elif kind == 2:
                rpg = 48
                addend = int_vec(g, -(-M // rpg), N)
            run_linear(f"linear {M}x{N}x{K}", a, w, bias=bias if j % 2 == 0 else None, addend=addend, rpg=rpg,
                       force_bn=bn)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("M", (1, 129, 257, 3952))
def test_linear_edges_bound(M, family):
    g = gen(M * 10 + FAMILIES.index(family))
    for i, N in enumerate(N_SWEEP):
        K = K_CYCLE[(i + M) % len(K_CYCLE)]
        a, w, bias = float_operands(family, g, M, N, K)
        for bn in bns_for(N)[::2] + [bns_for(N)[-1]]:
            run_linear(f"linear {M}x{N}x{K}", a, w, bias=bias, force_bn=bn, family=family,
                       signed=family == "all_positive")


@pytest.mark.parametrize("K", (64, 128, 192, 1024, 4096, 16384))
def test_linear_depth(K):
    """K from one k-block to 256 k-blocks, exact and under the bound (all-positive: the truncation model's worst case)."""
    g = gen(K)
    M, N = 257, 264
    run_linear(f"linear depth {M}x{N}x{K}", int_act(g, M, K), int_weight(g, N, K), bias=int_vec(g, N))
    for family in ("flat", "all_positive", "cancellation"):
        a, w, bias = float_operands(family, g, M, N, K)
        run_linear(f"linear depth {M}x{N}x{K}", a, w, bias=bias, family=family, signed=family == "all_positive")


@pytest.mark.parametrize("split", ("first", "middle", "last"))
def test_linear_k_split_strided(split):
    """The dual-source A (the 1x1 shortcut on concat(h, skip)): k_split at the first and last 64-boundary and between,
    a and a2 column slices of wider buffers (their own leading dimensions)."""
    g = gen(len(split))
    M, N, K = 1000, 320, 640
    k1 = {"first": 64, "middle": 320, "last": K - 64}[split]
    buf1, buf2 = int_act(g, M, k1 + 72), int_act(g, M, K - k1 + 136)
    a, a2 = buf1[:, 8:8 + k1], buf2[:, 64:64 + K - k1]
    w, bias = int_weight(g, N, K), int_vec(g, N)
    run_linear(f"linear dual source k_split {k1}", a, w, bias=bias, a2=a2)
    fa, fw, fb = float_operands("cancellation", g, M, N, K)
    fb1, fb2 = torch.zeros(M, k1 + 72, dtype=torch.float16, device=dev), torch.zeros(M, K - k1 + 136,
                                                                                      dtype=torch.float16, device=dev)
    fb1[:, 8:8 + k1], fb2[:, 64:64 + K - k1] = fa[:, :k1], fa[:, k1:]
    run_linear(f"linear dual source k_split {k1}", fb1[:, 8:8 + k1], fw, bias=fb, a2=fb2[:, 64:64 + K - k1],
               family="cancellation")


ADDEND_CASES = [("residual", 1), ("temb_staged", 256), ("temb_rows", 48), ("temb_rows", 127), ("temb_rows", 129)]


@pytest.mark.parametrize("mode,rpg", ADDEND_CASES)
@pytest.mark.parametrize("M,N,K", [(1000, 200, 192), (3952, 640, 640), (300, 1280, 320)])
def test_linear_addend_modes(M, N, K, mode, rpg):
    """Every addend mode, each also as a column slice of a wider buffer (ld_add != N, like the time-embedding slice of
    all resnets), exact and under the bound; the residual also in place. rpg = 127 / 129 put a sample boundary at the
    last / first row of a tile."""
    g = gen(M + N + rpg)
    a, w, bias = int_act(g, M, K), int_weight(g, N, K), int_vec(g, N)
    rows = M if rpg == 1 else -(-M // rpg)
    wide = int_vec(g, rows, N + 64)
    for addend in (int_vec(g, rows, N), wide[:, 32:32 + N]):
        run_linear(f"linear {M}x{N}x{K} ld_add {addend.stride(0)}", a, w, bias=bias, addend=addend, rpg=rpg)
    if rpg == 1:
        run_linear(f"linear {M}x{N}x{K}", a, w, bias=bias, addend=int_vec(g, M, N), in_place=True)
    fa, fw, fb = float_operands("flat", g, M, N, K)
    fad = torch.randn(rows, N + 64, generator=g, device=dev).half()[:, 16:16 + N]
    run_linear(f"linear {M}x{N}x{K} ld_add {fad.stride(0)}", fa, fw, bias=fb, addend=fad, rpg=rpg, family="flat")
    if rpg == 1:
        run_linear(f"linear {M}x{N}x{K}", fa, fw, bias=fb, addend=torch.randn(M, N, generator=g, device=dev).half(),
                   in_place=True, family="flat")


def test_linear_subnormal_and_overflow():
    """W·2^-24 (every output a multiple of 2^-24 below 2^-13: fp16 subnormals, exact), and a bias of ±65472 that puts
    the outputs across ±65504: overflow to ±inf exactly as .half() rounds."""
    g = gen(5)
    for M, N, K, bn in [(257, 264, 640, 0), (1000, 1280, 1280, 128), (77, 64, 2048, 64)]:
        a, w = int_act(g, M, K), int_weight(g, N, K)
        run_linear(f"linear subnormal {M}x{N}x{K}", a, (w.float() * 2.0 ** -24).half(), force_bn=bn)
        big = torch.where(torch.arange(N, device=dev) % 2 == 0, 65472.0, -65472.0).half()
        out = run_linear_overflow(a, w, big, bn)
        assert torch.isinf(out).any() and torch.isfinite(out).any(), "the outputs do not straddle the fp16 range"


def run_linear_overflow(a, w, bias, bn):
    from cfgpp_b200 import _native as nv
    out = nv.op_linear(a, w, bias, force_bn=bn)
    check_exact(f"linear overflow {a.shape[0]}x{w.shape[0]}x{w.shape[1]}", out, linear_kblocks(a), w, a.shape[0],
                bias, finite=False)
    return out


def geglu_int_operands(g, M, C):
    """GEGLU operands with exact value pre-activations |v| < 64 + 16 and gate pre-activations in [8, 136]."""
    inner = 4 * C
    a = int_act(g, M, C)
    w = int_weight(g, 2 * inner, C, nnz=15)
    bias = torch.cat([int_vec(g, inner), torch.full((inner,), 72.0, device=dev).half()])
    from test_gpu_gemm_epilogues import pack_geglu
    wp, bp = pack_geglu(w, bias)
    gates = ((a.float() @ w[inner:].float().t()) + 72.0)
    assert gates.min() >= 8, "a gate pre-activation below 8"
    assert_gelu_identity(gates)
    return a, wp, bp


@pytest.mark.parametrize("force_streamk", [False, True])
@pytest.mark.parametrize("M,C", [(77, 320), (1000, 640), (4096, 640), (3952, 1280)])
def test_geglu(M, C, force_streamk):
    """ff.net.0's GEGLU: exact with every gate g >= 8 (fp16(gelu(g)) = g), so out = fp16(fp16(a)·fp16(g)) pins the
    value / gate pairing of the packing; and flat inputs under the bound."""
    from test_gpu_gemm_epilogues import pack_geglu
    g = gen(M + C)
    a, wp, bp = geglu_int_operands(g, M, C)
    run_linear(f"geglu {M}x{4 * C}x{C}", a, wp, bias=bp, geglu=True, force_streamk=force_streamk)
    fa, fw, fb = float_operands("flat", g, M, 8 * C, C)
    fwp, fbp = pack_geglu(fw, fb)
    run_linear(f"geglu {M}x{4 * C}x{C}", fa, fwp, bias=fbp, geglu=True, force_streamk=force_streamk, family="flat")


# ================================================================================================= stream-K

@pytest.mark.parametrize("M,N,K", [(4096, 1280, 1280), (2048, 640, 2560), (5000, 1280, 640), (1000, 1280, 10240)])
def test_linear_streamk_forced(M, N, K):
    """The forced split feeds the plain epilogue: exact, and the cancellation family (large parked partials, small
    outputs) under the bound."""
    g = gen(M + N + K)
    res = int_vec(g, M, N)
    run_linear(f"linear {M}x{N}x{K}", int_act(g, M, K), int_weight(g, N, K), bias=int_vec(g, N), addend=res,
               force_streamk=True, expect_sk=True)
    for family in ("cancellation", "all_positive"):
        a, w, bias = float_operands(family, g, M, N, K)
        run_linear(f"linear {M}x{N}x{K}", a, w, bias=bias, force_streamk=True, expect_sk=True, family=family,
                   signed=family == "all_positive")


def test_streamk_three_pieces():
    """Fewer tiles than CTAs with a long K: every tile is split over >= 3 CTAs (the fix-up sums two or more parked
    partials), natural (convolution) and forced (linear)."""
    g = gen(3)
    x, w = int_act(g, 8, 8, 8, 1280), int_weight(g, 1280, 9 * 1280)
    run_conv("conv 8x8x8 1280->1280", x, w, bias=int_vec(g, 1280), expect_sk=True, pieces3=True)
    fx = torch.randn(8, 8, 8, 1280, generator=g, device=dev).add(100).half()
    fw = torch.randn(1280, 9 * 1280, generator=g, device=dev).mul((9 * 1280) ** -0.5)
    run_conv("conv 8x8x8 1280->1280", fx, (fw - fw.mean(1, keepdim=True)).half(), expect_sk=True, pieces3=True,
             family="cancellation")
    a, wl = int_act(g, 512, 8192), int_weight(g, 1280, 8192)
    run_linear("linear 512x1280x8192", a, wl, force_streamk=True, expect_sk=True, pieces3=True)
    fa, fwl, fb = float_operands("cancellation", g, 512, 1280, 8192)
    run_linear("linear 512x1280x8192", fa, fwl, bias=fb, force_streamk=True, expect_sk=True, pieces3=True,
               family="cancellation")


def test_streamk_repeatable():
    """Ten launches of a stream-K shape (natural conv, forced linear) are bit-identical."""
    from cfgpp_b200 import _native as nv
    g = gen(10)
    x, w, b = int_act(g, 2, 13, 19, 1280), int_weight(g, 1280, 9 * 1280), int_vec(g, 1280)
    assert nv.conv3x3_schedule(x, w, b)["streamk"]
    first = nv.op_conv3x3_ex(x, w, b)
    for _ in range(10):
        assert torch.equal(nv.op_conv3x3_ex(x, w, b), first)
    a, wl, bl = float_operands("flat", g, 4096, 1280, 1280)
    first = nv.op_linear(a, wl, bl, force_streamk=True)
    for _ in range(10):
        assert torch.equal(nv.op_linear(a, wl, bl, force_streamk=True), first)


# ================================================================================================= edge sweep: conv

CONV_EDGES = [  # B, H, W, Cin, Cout, stride, pad
    (1, 5, 7, 64, 64, 1, 1),        # one tile holds the whole image and runs past the batch
    (3, 11, 13, 128, 64, 1, 1),     # H·W = 143: tiles straddle images mid-row
    (16, 13, 13, 64, 72, 1, 1),     # B·H·W = 2704 = 21·128 + 16: the last tile walks past the last image
    (2, 8, 8, 128, 128, 1, 1),      # images smaller than a tile (tiled: two images per tile)
    (2, 32, 32, 64, 200, 1, 1),
    (2, 10, 14, 64, 64, 2, 1), (3, 24, 20, 64, 64, 2, 0), (2, 6, 10, 64, 64, 2, 0), (1, 16, 16, 64, 64, 2, 1),
    (2, 64, 64, 128, 128, 2, 0),
]


@pytest.mark.parametrize("im2col", [False, True])
@pytest.mark.parametrize("B,H,W,Cin,Cout,stride,pad", CONV_EDGES)
def test_conv_edges(B, H, W, Cin, Cout, stride, pad, im2col):
    """Both A-tile modes (where the tiled box can address the geometry), every stride / pad, temb per image, exact and
    under the bound (flat and dynamic range)."""
    from cfgpp_b200 import _native as nv
    g = gen(B * 1000 + H * 7 + W + Cin + stride + pad)
    x, w = int_act(g, B, H, W, Cin), int_weight(g, Cout, 9 * Cin)
    Ho, Wo = H // stride, W // stride
    tiled_ok = nv.conv3x3_schedule(x, w, stride=stride, pad=pad)["a_mode"] == "tiled"
    if not im2col and not tiled_ok:
        pytest.skip("only the im2col A tile addresses this geometry (covered by the im2col case)")
    temb = int_vec(g, B, Cout)
    for addend, rpg in ((None, 1), (temb, Ho * Wo), (int_vec(g, B * Ho * Wo, Cout), 1)):
        run_conv(f"conv {B}x{H}x{W} {Cin}->{Cout}", x, w, bias=int_vec(g, Cout), addend=addend, rpg=rpg,
                 stride=stride, pad=pad, force_im2col=im2col, expect_mode="im2col" if im2col else "tiled")
    for family in ("flat", "dynamic_range"):
        fx, fw, fb = float_operands(family, g, B * H * W, Cout, 9 * Cin)
        fx = fx[:, :Cin].reshape(B, H, W, Cin).contiguous()
        run_conv(f"conv {B}x{H}x{W} {Cin}->{Cout}", fx, fw, bias=fb, addend=temb.float().mul(0.1).half(),
                 rpg=Ho * Wo, stride=stride, pad=pad, force_im2col=im2col, family=family)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 8, 8, 128, 128), (4, 32, 32, 320, 320), (1, 40, 256, 64, 64)])
def test_conv_force_bn(B, H, W, Cin, Cout):
    """Every tile width on a convolution, exact."""
    g = gen(B + H + Cin)
    x, w, b = int_act(g, B, H, W, Cin), int_weight(g, Cout, 9 * Cin), int_vec(g, Cout)
    for bn in bns_for(Cout):
        run_conv(f"conv {B}x{H}x{W} {Cin}->{Cout}", x, w, bias=b, force_bn=bn)


# ================================================================================================= moved cases
# the GEMM / conv cases of the former rel-L2 suite, every parameter set, now under the per-element bound

@pytest.mark.parametrize("M,N,K,hb,ha,bn", [
    (128, 64, 64, False, 0, 64), (256, 256, 256, True, 0, 256), (256, 320, 320, True, 1, 160),
    (308, 1280, 2048, False, 0, 0), (4096, 1280, 1280, True, 1, 0), (2048, 320, 960, True, 1024, 0),
    (1000, 200, 192, True, 1, 128), (16384, 1920, 640, False, 0, 0), (1, 64, 64, True, 0, 0), (77, 8, 64, False, 0, 0)])
def test_linear(M, N, K, hb, ha, bn):
    g = torch.Generator().manual_seed(M * 7 + N)
    a, w = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5)
    bias = rnd(g, N) if hb else None
    addend = rnd(g, M, N) if ha == 1 else (rnd(g, (M + ha - 1) // ha, N) if ha > 1 else None)
    run_linear(f"linear {M}x{N}x{K}", a, w, bias=bias, addend=addend, rpg=ha if ha > 1 else 1, force_bn=bn,
               family="flat")


@pytest.mark.parametrize("force_streamk", [False, True])
@pytest.mark.parametrize("M,N,K,geglu_like", [(4096, 1280, 1280, False), (4096, 1280, 5120, False),
                                              (4096, 3840, 1280, False), (2048, 640, 2560, False),
                                              (8192, 1280, 1280, False), (5000, 1280, 640, False)])
def test_linear_streamk_shapes_and_repeatability(M, N, K, geglu_like, force_streamk):
    """Shapes whose tile count is not a multiple of the CTA count: the linear layers skip the stream-K split unless
    `force_streamk` is set (asserted through the schedule). Result under the bound, 12 launches bit-identical."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(M + N + K)
    a, w, bias, res = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5), rnd(g, N), rnd(g, M, N)
    if not nv.linear_schedule(a, w, bias, res, force_streamk=True)["streamk"]:
        pytest.skip("the tiles fill whole rounds over this card's SMs: no remainder to split")
    first, _ = run_linear(f"linear {M}x{N}x{K}", a, w, bias=bias, addend=res, force_streamk=force_streamk,
                          expect_sk=force_streamk, family="flat")
    for _ in range(12):
        assert torch.equal(nv.op_linear(a, w, bias, res, 1, force_streamk=force_streamk), first)


def test_linear_dual_source_and_geglu():
    from test_gpu_gemm_epilogues import pack_geglu
    g = torch.Generator().manual_seed(5)
    a1, a2 = rnd(g, 1024, 640), rnd(g, 1024, 320)
    w, bias = rnd(g, 320, 960, scale=960 ** -0.5), rnd(g, 320)
    run_linear("linear dual-source", a1, w, bias=bias, a2=a2, family="flat")
    M, Cc = 512, 640
    a, w, b = rnd(g, M, Cc), rnd(g, 8 * Cc, Cc, scale=Cc ** -0.5), rnd(g, 8 * Cc)
    wp, bp = pack_geglu(w, b)
    run_linear("geglu", a, wp, bias=bp, geglu=True, family="flat")


def nchw_case(g, B, Cin, H, W, Cout):
    x, w, bias = rnd(g, B, Cin, H, W), rnd(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5), rnd(g, Cout)
    return x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous(), bias


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(4, 128, 128, 320, 320), (4, 64, 64, 640, 640), (2, 32, 32, 128, 128),
                                            (1, 16, 16, 64, 64), (2, 96, 128, 64, 64)])
def test_conv3x3_stride2(B, H, W, Cin, Cout):
    """Downsample2D (3x3, stride 2, pad 1): the first row / column of taps starts at input coordinate -1 (zero fill),
    every second pixel is fetched."""
    g = torch.Generator().manual_seed(H + Cin)
    x, w, bias = nchw_case(g, B, Cin, H, W, Cout)
    run_conv(f"conv {B}x{H}x{W} {Cin}->{Cout}", x, w, bias=bias, stride=2, pad=1, family="flat")


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 256, 256, 128, 128), (2, 128, 128, 256, 256), (2, 32, 32, 64, 64),
                                            (1, 64, 128, 128, 128)])
def test_conv3x3_stride2_pad_after(B, H, W, Cin, Cout):
    """The AutoencoderKL encoder's Downsample2D: one zero row / column after the image, then an un-padded stride-2
    conv."""
    g = torch.Generator().manual_seed(H + Cin + 1)
    x, w, bias = nchw_case(g, B, Cin, H, W, Cout)
    run_conv(f"conv {B}x{H}x{W} {Cin}->{Cout}", x, w, bias=bias, stride=2, pad=0, family="flat")


def test_conv3x3_streamk_repeatable():
    """The conv shapes of the 1280-channel level take the stream-K split by default: 10 launches, bit-identical."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(11)
    x, w, bias = rnd(g, 4, 32, 32, 1280), rnd(g, 1280, 9 * 1280, scale=(9 * 1280) ** -0.5), rnd(g, 1280)
    res = rnd(g, 4 * 32 * 32, 1280)
    first, _ = run_conv("conv 4x32x32 1280->1280", x, w, bias=bias, addend=res, family="flat", expect_sk=True)
    for _ in range(10):
        assert torch.equal(nv.op_conv3x3(x, w, bias, res, 1).reshape(first.shape), first)


@pytest.mark.parametrize("B,H,W,Cin,Cout,ht,hr", [
    (1, 32, 32, 64, 64, False, False), (2, 64, 64, 128, 128, True, False), (4, 16, 16, 128, 256, False, True),
    (2, 8, 8, 128, 128, True, False), (1, 128, 128, 320, 320, True, False), (4, 32, 32, 1280, 1280, False, True),
    (2, 96, 128, 64, 128, True, False), (1, 24, 32, 128, 128, False, True), (3, 6, 64, 64, 64, False, False),
    (1, 40, 256, 64, 64, False, True), (1, 16, 1024, 64, 64, True, False),
    (8, 8, 8, 1280, 1280, True, False), (8, 8, 8, 2560, 1280, False, True)])
def test_conv3x3(B, H, W, Cin, Cout, ht, hr):
    """Zero padding comes from the TMA's out-of-bounds fill: every element gated, edge pixels included."""
    g = torch.Generator().manual_seed(H * 3 + Cin)
    xn, w, bias = rnd(g, B, Cin, H, W), rnd(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5), rnd(g, Cout)
    addend, rpg = None, 1
    if ht:
        addend, rpg = rnd(g, B, Cout), H * W
    elif hr:
        addend = rnd(g, B * H * W, Cout)
    x, wp = xn.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    run_conv(f"conv {B}x{H}x{W} {Cin}->{Cout}", x, wp, bias=bias, addend=addend, rpg=rpg, family="flat")


# ================================================================================================= invariances

def test_batch_equals_images():
    """A batch equals its images run one by one (conv and linear rows alike), where the schedule shows the same tile
    width and no stream-K on both sides."""
    from cfgpp_b200 import _native as nv
    g = gen(21)
    for B, H, W, C in [(4, 16, 16, 128), (3, 11, 13, 64), (2, 64, 64, 320)]:
        x, w, b = torch.randn(B, H, W, C, generator=g, device=dev).half(), int_weight(g, C, 9 * C), int_vec(g, C)
        full_s = nv.conv3x3_schedule(x, w, b)
        full = nv.op_conv3x3_ex(x, w, b)
        for i in range(B):
            xi = x[i:i + 1].contiguous()
            s = nv.conv3x3_schedule(xi, w, b, force_bn=full_s["bn"])
            if full_s["streamk"] or s["streamk"]:
                continue
            assert torch.equal(nv.op_conv3x3_ex(xi, w, b, force_bn=full_s["bn"]), full[i:i + 1]), f"conv image {i}"
    a, wl, bl = float_operands("flat", g, 1000, 640, 640)
    full = nv.op_linear(a, wl, bl, force_bn=128)
    for r0, r1 in [(0, 128), (128, 300), (999, 1000), (500, 1000)]:
        assert torch.equal(nv.op_linear(a[r0:r1].contiguous(), wl, bl, force_bn=128), full[r0:r1]), f"rows {r0}:{r1}"


# ================================================================================================= production launches

def unet_gemm_launches(cfg, h, w, NB=4):
    """Every GEMM / conv launch of a UNet's body and tail plans (plus the prompt plan's to_kv) on an h x w latent at
    UNet batch NB, in the order `Unet::prepare` builds them: dicts with the plan name, kind ('conv' / 'linear'),
    algorithmic FLOPs and the production layout."""
    ch, L, lpb = cfg.block_out_channels, len(cfg.block_out_channels), cfg.layers_per_block
    D, n_ctx = cfg.cross_attention_dim, 77
    down_attn = [t.startswith("CrossAttn") for t in cfg.down_block_types]
    up_attn = [t.startswith("CrossAttn") for t in cfg.up_block_types]
    order = [(f"down_blocks.{i}.resnets.{j}", ch[i]) for i in range(L) for j in range(lpb)]
    order += [("mid_block.resnets.0", ch[-1]), ("mid_block.resnets.1", ch[-1])]
    order += [(f"up_blocks.{i}.resnets.{j}", ch[L - 1 - i]) for i in range(L) for j in range(lpb + 1)]
    temb_off, tot = {}, 0
    for name, c in order:
        temb_off[name] = tot
        tot += c
    out = []

    def conv(name, H, W, Cin, Cout, stride=1, **lay):
        Ho, Wo = H // stride, W // stride
        out.append(dict(name=name, kind="conv", B=NB, H=H, W=W, Cin=Cin, Cout=Cout, stride=stride, pad=1,
                        flops=2.0 * NB * Ho * Wo * Cout * 9 * Cin, **lay))

    def lin(name, M, N, K, flops=None, **lay):
        out.append(dict(name=name, kind="linear", M=M, N=N, K=K, flops=2.0 * M * N * K if flops is None else flops,
                        **lay))

    def resnet(p, C1, C2, Cout, H, W):
        Cin = C1 + C2
        conv(p + ".conv1", H, W, Cin, Cout, addend="temb", ld_add=tot, temb_off=temb_off[p])
        if Cin != Cout:
            lin(p + ".conv_shortcut", NB * H * W, Cout, Cin, k_split=C1)
        conv(p + ".conv2", H, W, Cout, Cout, addend="residual")

    def transformer(p, C, H, W, layers, heads):
        M = NB * H * W
        hdp = -(-(C // heads) // 64) * 64
        Cp = heads * hdp
        lin(p + ".proj_in", M, C, C)
        for k in range(layers):
            b = f"{p}.transformer_blocks.{k}"
            lin(b + ".attn1.to_qkv(+norm1)", M, 3 * Cp, C, flops=2.0 * M * 3 * C * C, bias=False)
            lin(b + ".attn1.to_out", M, C, Cp, flops=2.0 * M * C * C, addend="in_place")
            lin(b + ".attn2.to_q(+norm2)", M, Cp, C, flops=2.0 * M * C * C, bias=False)
            lin(b + ".attn2.to_kv", NB * n_ctx, 2 * Cp, D, flops=2.0 * NB * n_ctx * 2 * C * D, bias=False, plan="prompt")
            lin(b + ".attn2.to_out", M, C, Cp, flops=2.0 * M * C * C, addend="in_place")
            lin(b + ".ff.geglu(+norm3)", M, 8 * C, C, geglu=True)
            lin(b + ".ff.out", M, C, 4 * C, addend="in_place")
        lin(p + ".proj_out", M, C, C, addend="residual")

    H, W, cur, skips = h, w, ch[0], [ch[0]]
    for i in range(L):
        for j in range(lpb):
            resnet(f"down_blocks.{i}.resnets.{j}", cur, 0, ch[i], H, W)
            cur = ch[i]
            if down_attn[i]:
                transformer(f"down_blocks.{i}.attentions.{j}", cur, H, W, cfg.transformer_layers_per_block[i],
                            cfg.num_attention_heads[i])
            skips.append(cur)
        if i != L - 1:
            conv(f"down_blocks.{i}.downsamplers.0.conv", H, W, cur, cur, stride=2)
            H, W = H // 2, W // 2
            skips.append(cur)
    resnet("mid_block.resnets.0", cur, 0, cur, H, W)
    transformer("mid_block.attentions.0", cur, H, W, cfg.transformer_layers_per_block[-1], cfg.num_attention_heads[-1])
    resnet("mid_block.resnets.1", cur, 0, cur, H, W)
    for i in range(L):
        rev = L - 1 - i
        for j in range(lpb + 1):
            resnet(f"up_blocks.{i}.resnets.{j}", cur, skips.pop(), ch[rev], H, W)
            cur = ch[rev]
            if up_attn[i]:
                transformer(f"up_blocks.{i}.attentions.{j}", cur, H, W, cfg.transformer_layers_per_block[rev],
                            cfg.num_attention_heads[rev])
        if i != L - 1:
            conv(f"up_blocks.{i}.upsamplers.0.conv", 2 * H, 2 * W, cur, cur)
            H, W = 2 * H, 2 * W
    assert not skips and (H, W) == (h, w)
    return out


def vae_gemm_launches(cfg, H, W):
    """Every GEMM / conv launch of the AutoencoderKL decoder (latent H/8 x W/8) and encoder (H x W image), batch 1."""
    ch, L, lpb = cfg.block_out_channels, len(cfg.block_out_channels), cfg.layers_per_block
    out = []

    def conv(part, h, w, Cin, Cout, stride=1, pad=1, **lay):
        out.append(dict(name=part, kind="conv", B=1, H=h, W=w, Cin=Cin, Cout=Cout, stride=stride, pad=pad, **lay))

    def lin(part, M, N, K, **lay):
        out.append(dict(name=part, kind="linear", M=M, N=N, K=K, **lay))

    def resnet(part, Cin, Cout, h, w):
        conv(part + " resnet.conv1", h, w, Cin, Cout)
        if Cin != Cout:
            lin(part + " resnet.conv_shortcut", h * w, Cout, Cin)
        conv(part + " resnet.conv2", h, w, Cout, Cout, addend="residual")

    def attention(part, C, h, w):
        n = h * w
        lin(part + " attn.to_q", n, C, C)
        lin(part + " attn.to_k", n, C, C)
        lin(part + " attn.QK^T", n, n, C, bias=False)
        lin(part + " attn.V0^T=Wv.X^T", C, n, C, bias=False)
        lin(part + " attn.P.V0+b_v", n, C, n, softmax=True)
        lin(part + " attn.to_out", n, C, C, addend="residual")

    f = 1 << (L - 1)
    h, w, C = H // f, W // f, ch[-1]
    resnet("decoder mid", C, C, h, w)
    attention("decoder mid", C, h, w)
    resnet("decoder mid", C, C, h, w)
    for i in range(L):
        Cout = ch[L - 1 - i]
        for _ in range(lpb + 1):
            resnet(f"decoder up{i}", C, Cout, h, w)
            C = Cout
        if i != L - 1:
            h, w = 2 * h, 2 * w
            conv(f"decoder up{i} upsample", h, w, C, C)
    h, w, C = H, W, ch[0]
    for i in range(L):
        for _ in range(lpb):
            resnet(f"encoder down{i}", C, ch[i], h, w)
            C = ch[i]
        if i != L - 1:
            conv(f"encoder down{i} downsample", h, w, C, C, stride=2, pad=0)
            h, w = h // 2, w // 2
    resnet("encoder mid", C, C, h, w)
    attention("encoder mid", C, h, w)
    resnet("encoder mid", C, C, h, w)
    return out


def clip_gemm_launches(cfg, B):
    M, D, I = 77 * B, cfg.hidden_size, cfg.intermediate_size
    return [dict(name=f"{cfg.name} qkv", kind="linear", M=M, N=3 * D, K=D),
            dict(name=f"{cfg.name} out_proj", kind="linear", M=M, N=D, K=D, addend="residual"),
            dict(name=f"{cfg.name} fc1", kind="linear", M=M, N=I, K=D),
            dict(name=f"{cfg.name} fc2", kind="linear", M=M, N=D, K=I, addend="residual")]


# layout keys of the ControlNet and vision-tower launches: the real channel counts of a zero-padded convolution, the
# real K of the patch GEMM, the (heads, head_dim) of head-padded q|k|v rows or out_proj columns
EXTRA_KEYS = ("cin_real", "cout_real", "k_real", "vit_heads", "ip_heads")


def pad64(c):
    return -(-c // 64) * 64


def controlnet_body_launches(cfg, h, w, NB=4):
    """The GEMM / conv launches of a ControlNet's body (its down blocks and mid block, the UNet's shapes) on an h x w
    latent: `unet_gemm_launches` without the up path, the tail and the prompt plan, and with the time-embedding rows of
    the ControlNet's own resnets (down and mid only), so the temb row stride is the ControlNet's."""
    ch, L, lpb = cfg.block_out_channels, len(cfg.block_out_channels), cfg.layers_per_block
    order = [f"down_blocks.{i}.resnets.{j}" for i in range(L) for j in range(lpb)]
    order += ["mid_block.resnets.0", "mid_block.resnets.1"]
    widths = [ch[i] for i in range(L) for _ in range(lpb)] + [ch[-1], ch[-1]]
    off, tot = {}, 0
    for n, c in zip(order, widths):
        off[n] = tot
        tot += c
    out = []
    for l in unet_gemm_launches(cfg, h, w, NB):
        if l.get("plan") == "prompt" or not l["name"].startswith(("down_blocks.", "mid_block.")):
            continue
        l = dict(l)
        if l.get("addend") == "temb":
            l.update(ld_add=tot, temb_off=off[l["name"].rsplit(".", 1)[0]])
        out.append(l)
    return out


def controlnet_embed_launches(cn_cfg, h, w, B):
    """The conditioning embedding's convolutions on B images of 8h x 8w, as `Unet::cond_embed` issues them: NHWC
    activations and weights with the channels zero-padded to whole 64-wide K blocks (`packed_conv3x3`), stride 2
    with pad 1 on blocks.1 / 3 / 5, conv_out to the unpadded C0."""
    ch, C0 = cn_cfg.conditioning_embedding_out_channels, cn_cfg.unet.block_out_channels[0]
    H, W, out = 8 * h, 8 * w, []

    def conv(name, cin, cout, cout_p, stride):
        nonlocal H, W
        out.append(dict(name=f"controlnet_cond_embedding.{name}", kind="conv", B=B, H=H, W=W, Cin=pad64(cin),
                        Cout=cout_p, stride=stride, pad=1, cin_real=cin, cout_real=cout,
                        flops=2.0 * B * (H // stride) * (W // stride) * cout * 9 * cin))
        H, W = H // stride, W // stride

    conv("conv_in", cn_cfg.conditioning_channels, ch[0], pad64(ch[0]), 1)
    for i in range(len(ch) - 1):
        conv(f"blocks.{2 * i}", ch[i], ch[i], pad64(ch[i]), 1)
        conv(f"blocks.{2 * i + 1}", ch[i], ch[i + 1], pad64(ch[i + 1]), 2)
    conv("conv_out", ch[-1], C0, C0, 1)
    assert (H, W) == (h, w)
    return out


def t2i_adapter_gemm_launches(cfg, H, W, B):
    """The GEMM / conv launches of a T2I-Adapter (`t2i_adapter.T2IAdapterConfig`) on B images of H x W, as
    `T2IAdapter::prepare` issues them: conv_in, a 3x3 conv over the pixel-unshuffled image (Cin = in_channels·f²);
    per block, after the 2x2 pool of a down block, in_conv (a 1x1 conv as a linear) where the width changes, then per
    resnet block1 (3x3 conv) and block2 (1x1 linear with the residual added in place). Names are the weights'
    `adapter.*` keys; FLOPs 2·M·N·K, as `GemmOp::flops` counts them."""
    f = cfg.downscale_factor
    h, w, out = H // f, W // f, []

    def conv(name, cin, cout):
        out.append(dict(name=name, kind="conv", B=B, H=h, W=w, Cin=cin, Cout=cout, stride=1, pad=1,
                        flops=2.0 * B * h * w * cout * 9 * cin))

    def lin(name, N, K, **lay):
        M = B * h * w
        out.append(dict(name=name, kind="linear", M=M, N=N, K=K, flops=2.0 * M * N * K, **lay))

    conv("adapter.conv_in", cfg.in_channels * f * f, cfg.channels[0])
    for i, (cin, cout, down) in enumerate(cfg.blocks()):
        p = f"adapter.body.{i}"
        if down:
            h, w = h // 2, w // 2
        if cin != cout:
            lin(f"{p}.in_conv", cout, cin)
        for j in range(cfg.num_res_blocks):
            conv(f"{p}.resnets.{j}.block1", cout, cout)
            lin(f"{p}.resnets.{j}.block2", cout, cout, addend="in_place")
    assert cfg.feature_shapes(H, W)[-1] == (cfg.channels[-1], h, w)
    return out


def zero_conv_launches(cn_cfg, h, w, NB=4):
    """The zero convs of `Unet::build_control_plan`: per ControlNet residual k (`residual_channels` order, the last one
    the mid block's) a 1x1 convolution as a linear over the residual's NB·HW rows, N = K = C, with the scaled-residual
    epilogue in place into the UNet's skip tensor."""
    ch, L, lpb = cn_cfg.unet.block_out_channels, len(cn_cfg.unet.block_out_channels), cn_cfg.unet.layers_per_block
    H, W, hw = h, w, [h * w]
    for i in range(L):
        hw += [H * W] * lpb
        if i != L - 1:
            H, W = H // 2, W // 2
            hw.append(H * W)
    hw.append(H * W)
    res = cn_cfg.residual_channels
    assert len(res) == len(hw)
    names = [f"controlnet_down_blocks.{k}" for k in range(len(res) - 1)] + ["controlnet_mid_block"]
    return [dict(name=n, kind="linear", M=NB * p, N=C, K=C, addend="scaled_residual", flops=2.0 * NB * p * C * C)
            for n, C, p in zip(names, res, hw)]


def vision_gemm_launches(vcfg, tower, B):
    """The vision tower's GEMMs at B images, as `ClipVisionEncoder::encode` and `build_clip_layers` issue them: the
    patch GEMM (K = 3·P² zero-padded to whole k blocks, no bias), q|k|v into heads zero-padded to 64-multiples
    (N = 3·Cp, bias), out_proj over the padded head columns (K = Cp, residual), fc1, fc2 (residual)."""
    D, I, H, P = vcfg.hidden_size, vcfg.intermediate_size, vcfg.num_attention_heads, vcfg.patch_size
    hd = D // H
    Cp, K = H * pad64(hd), 3 * P * P
    npch = (vcfg.image_size // P) ** 2
    M = B * (npch + 1)
    return [dict(name=f"{tower} patch_embedding", kind="linear", M=B * npch, N=D, K=pad64(K), bias=False, k_real=K),
            dict(name=f"{tower} qkv", kind="linear", M=M, N=3 * Cp, K=D, vit_heads=(H, hd)),
            dict(name=f"{tower} out_proj", kind="linear", M=M, N=D, K=Cp, addend="residual", vit_heads=(H, hd)),
            dict(name=f"{tower} fc1", kind="linear", M=M, N=I, K=D),
            dict(name=f"{tower} fc2", kind="linear", M=M, N=D, K=I, addend="residual")]


def resampler_gemm_launches(g, D, T, NB):
    """The GEMMs of an IP-Adapter Plus Resampler of geometry g (`ip_adapter.plus_geometry`) giving D-wide tokens, on
    NB rows of T hidden states, as `Unet::build_ip_resampler` issues them (layer 0 stands for all: the layers share
    their shapes): proj_in, per layer to_q, to_kv over the hidden states and the latents, to_out and the feed-forward
    (in place into the latents), then proj_out. Names are the weights' `image_proj.*` keys."""
    Q, E, dim, inner, F = g["num_queries"], g["embed_dim"], g["dim"], 64 * g["heads"], g["ff_mult"] * g["dim"]
    lin = lambda n, M, N, K, **kw: dict(name="image_proj." + n, kind="linear", M=M, N=N, K=K, **kw)  # noqa: E731
    return [lin("proj_in", NB * T, dim, E), lin("layers.0.0.to_q", NB * Q, inner, dim, bias=False),
            lin("layers.0.0.to_kv", NB * (T + Q), 2 * inner, dim, bias=False),
            lin("layers.0.0.to_out", NB * Q, dim, inner, bias=False, addend="in_place"),
            lin("layers.0.1.1", NB * Q, F, dim, bias=False),
            lin("layers.0.1.3", NB * Q, dim, F, bias=False, addend="in_place"),
            lin("proj_out", NB * Q, D, dim)]


def ip_adapter_gemm_launches(cfg, E, n_tokens, NB=4, resampler=False):
    """An IP-Adapter's GEMMs in the UNet's image plan at UNet batch NB: image_proj.proj (M = NB, N = n_tokens·D, K = E,
    bias), or with `resampler` the Plus adapter's Resampler (`plus_geometry(cfg, E)`, over the hidden states of the
    tower that E selects; n_tokens must be its num_queries), then per transformer block attn2.to_kv_ip
    (M = NB·n_tokens, N = 2·Cp over heads zero-padded to 64-multiples, K = D, no bias)."""
    import production as P
    D = cfg.cross_attention_dim
    if resampler:
        from cfgpp_b200 import ip_adapter as IP
        g = IP.plus_geometry(cfg, E)
        assert n_tokens == g["num_queries"], f"the Resampler gives {g['num_queries']} tokens, not {n_tokens}"
        out = resampler_gemm_launches(g, D, IP.plus_encoder_config(cfg, E).num_positions, NB)
    else:
        out = [dict(name="image_proj.proj", kind="linear", M=NB, N=n_tokens * D, K=E)]
    for l in P.unet_attn_launches(cfg, 8, 8):  # the block list does not depend on the latent size
        if l["name"].endswith(".attn2.sdpa"):
            H, hd = l["heads"], l["hd"]
            out.append(dict(name=l["name"][:-len(".sdpa")] + ".to_kv_ip", kind="linear", M=NB * n_tokens,
                            N=2 * H * pad64(hd), K=D, bias=False, ip_heads=(H, hd)))
    return out


def signature(l):
    keys = ("kind", "B", "H", "W", "Cin", "Cout", "stride", "pad", "M", "N", "K", "addend", "k_split", "geglu",
            "bias", "softmax", "ld_add")
    return tuple(l.get(k) for k in keys) + tuple((k, l[k]) for k in EXTRA_KEYS if k in l)


def unique_launches(launches):
    seen, out = set(), []
    for l in launches:
        s = signature(l)
        if s not in seen:
            seen.add(s)
            out.append(l)
    return out


def production_lists():
    """{(model, size): [(case id, launch)]} over `production.py`: each UNet at each latent size, the VAE at each image
    size, each text tower at each prompt batch, and the ControlNets, vision towers, IP-Adapters (plain and Plus) and
    T2I-Adapters. Launches are unique within a list, not across lists."""
    import production as P
    from cfgpp_b200 import config as C
    from cfgpp_b200.text_encoder import CLIP_CONFIGS
    from cfgpp_b200.vae import VAEConfig
    out = {}
    for m, h, w in P.unet_sizes():
        tag = P.size_tag(m, h, w)
        out[(m, (h, w))] = [(f"{tag}-{i}-{l['name']}", l)
                            for i, l in enumerate(unique_launches(unet_gemm_launches(C.CONFIGS[m](), h, w)))]
    for H, W in P.VAE_SIZES:
        out[("vae", (H, W))] = [(f"vae-{W}x{H}-{i}-{l['name']}", l)
                                for i, l in enumerate(unique_launches(vae_gemm_launches(VAEConfig(), H, W)))]
    for tower, batches in P.TEXT_TOWERS.items():
        for B in batches:
            out[(tower, B)] = [(f"B{B}-{l['name']}", l) for l in clip_gemm_launches(CLIP_CONFIGS[tower](), B)]
    out.update(controlnet_production_lists())
    for tower, batches in P.VISION_TOWERS.items():
        for B in batches:
            out[(tower, B)] = [(f"B{B}-{l['name']}", l) for l in vision_gemm_launches(P.vision_config(tower), tower, B)]
    for m, E in P.IP_ADAPTERS:
        out[("ip_adapter", m, E)] = [(f"ip-{m}-E{E}-{i}-{l['name']}", l) for i, l in
                                     enumerate(unique_launches(ip_adapter_gemm_launches(C.CONFIGS[m](), E, P.IP_TOKENS)))]
    out.update(adapter_production_lists())
    return out


def ip_plus_launches(m, E):
    """An IP-Adapter Plus's launches (`ip_adapter_gemm_launches` with the Resampler) at every UNet batch of
    IP_PLUS_NB, each name prefixed with its NB."""
    from cfgpp_b200 import config as C, ip_adapter as IP
    cfg = C.CONFIGS[m]()
    Q = IP.plus_geometry(cfg, E)["num_queries"]
    return [dict(l, name=f"NB{NB} {l['name']}") for NB in P.IP_PLUS_NB
            for l in ip_adapter_gemm_launches(cfg, E, Q, NB, resampler=True)]


def t2i_launches(m, h, w):
    """A T2I-Adapter's launches for the UNet m on an h x w latent (8h x 8w images) at every batch and image channel
    count of `production.py`, each name prefixed with them."""
    from cfgpp_b200 import config as C, t2i_adapter as T
    return [dict(l, name=f"B{B} C{ci} {l['name']}") for ci in P.T2I_IN_CHANNELS for B in P.T2I_ADAPTER_BATCHES
            for l in t2i_adapter_gemm_launches(T.t2i_adapter_config(C.CONFIGS[m](), ci), 8 * h, 8 * w, B)]


def adapter_production_lists():
    """{("ip_adapter_plus", model, E): [(case id, launch)]} over IP_PLUS_ADAPTERS and {("t2i_adapter", model, size):
    [(case id, launch)]} over T2I_ADAPTER_SIZES."""
    out = {}
    for m, E in P.IP_PLUS_ADAPTERS:
        out[("ip_adapter_plus", m, E)] = [(f"ip-plus-{m}-E{E}-{i}-{l['name']}", l)
                                          for i, l in enumerate(unique_launches(ip_plus_launches(m, E)))]
    for m, h, w in P.t2i_sizes():
        out[("t2i_adapter", m, (h, w))] = [(f"t2i-{P.size_tag(m, h, w)}-{i}-{l['name']}", l)
                                           for i, l in enumerate(unique_launches(t2i_launches(m, h, w)))]
    return out


def controlnet_production_lists():
    """{("controlnet", model, size): [(case id, launch)]}: per controlled model and latent size, the ControlNet body,
    the zero convs and the conditioning embedding at every image batch of CONTROL_IMAGE_BATCHES."""
    import production as P
    from cfgpp_b200 import config as C, controlnet as CN
    out = {}
    for m, h, w in P.controlnet_sizes():
        cfg = C.CONFIGS[m]()
        cn_cfg = CN.controlnet_config(cfg)
        launches = controlnet_body_launches(cfg, h, w) + zero_conv_launches(cn_cfg, h, w)
        for B in P.CONTROL_IMAGE_BATCHES:
            launches += [dict(l, name=f"B{B} {l['name']}") for l in controlnet_embed_launches(cn_cfg, h, w, B)]
        out[("controlnet", m, (h, w))] = [(f"cn-{P.size_tag(m, h, w)}-{i}-{l['name']}", l)
                                         for i, l in enumerate(unique_launches(launches))]
    return out


def _production_cases():
    """One case per launch signature over all production lists: a shape shared by two models or sizes (SD v1.5 and
    SD 2-base, the VAE at two sizes) runs once, under the id of the first list that has it."""
    seen, cases = set(), []
    for launches in production_lists().values():
        for cid, l in launches:
            if signature(l) not in seen:
                seen.add(signature(l))
                cases.append(pytest.param(l, id=cid))
    return cases


def run_production(l, family):
    """One production launch in its layout. family None: Family A (exact), else Family B."""
    from test_gpu_gemm_epilogues import pack_geglu
    g = gen(zlib.crc32(repr(signature(l)).encode()) + (family is not None))
    exact = family is None
    name = l["name"]
    if l["kind"] == "conv":
        B, H, W, Cin, Cout, s = l["B"], l["H"], l["W"], l["Cin"], l["Cout"], l["stride"]
        Mo = B * (H // s) * (W // s)
        if exact:
            x, w, b = int_act(g, B, H, W, Cin), int_weight(g, Cout, 9 * Cin), int_vec(g, Cout)
        else:
            x = torch.randn(B, H, W, Cin, generator=g, device=dev).half()
            w = (torch.randn(Cout, 9 * Cin, generator=g, device=dev) * (9 * Cin) ** -0.5).half()
            b = torch.randn(Cout, generator=g, device=dev).half()
        if "cin_real" in l:  # zero-padded channels: +0 inputs, zero weight rows / columns and bias entries
            ci, co = l["cin_real"], l["cout_real"]
            x[..., ci:] = 0
            w = w.reshape(Cout, 9, Cin)
            w[:, :, ci:] = 0
            w[co:] = 0
            w = w.reshape(Cout, 9 * Cin)
            b[co:] = 0
        addend, rpg = None, 1
        mk = (lambda *s: int_vec(g, *s)) if exact else (lambda *s: torch.randn(*s, generator=g, device=dev).half())
        if l.get("addend") == "temb":  # the resnet's column slice of the time-embedding rows of all resnets
            temb_all = mk(B, l["ld_add"])
            addend, rpg = temb_all[:, l["temb_off"]:l["temb_off"] + Cout], (H // s) * (W // s)
        elif l.get("addend") == "residual":
            addend = mk(Mo, Cout)
        out, sched = run_conv(name, x, w, bias=b, addend=addend, rpg=rpg, stride=s, pad=l["pad"], family=family)
        if " adapter." in name:  # a T2I-Adapter convolution: its A tile and image batch
            SEEN["t2i_conv"].add((sched["a_mode"], B))
        if "cout_real" in l:
            assert (out[:, l["cout_real"]:].view(torch.int16) == 0).all(), f"{name}: padded channels are not +0"
        return
    M, N, K = l["M"], l["N"], l["K"]
    geglu = bool(l.get("geglu"))
    if exact and geglu:
        a, w, b = geglu_int_operands(g, M, K)
    elif exact:
        a, w = int_act(g, M, K), int_weight(g, N, K)
        b = int_vec(g, N) if l.get("bias", True) else None
    else:
        a, w, b = float_operands("flat", g, M, N, K)
        if l.get("softmax"):  # P·V0 + b_v: fp16 softmax rows against V0 at mean 10σ
            a = softmax_rows(g, M, K, peaked=False)
            w = (torch.randn(N, K, generator=g, device=dev) + 10).half()
        if geglu:
            w, b = pack_geglu(w, b)
        if not l.get("bias", True):
            b = None
    if "k_real" in l:  # the patch GEMM: columns K_real..K-1 of A and W zero
        a[:, l["k_real"]:] = 0
        w[:, l["k_real"]:] = 0
    for key in ("vit_heads", "ip_heads"):
        if key in l:  # rows (q|k|v, K‖V) or columns (out_proj) of every head's padding zero
            H, hd = l[key]
            if K == H * pad64(hd):
                a[:, (torch.arange(K, device=dev) % pad64(hd)) >= hd] = 0
                w[:, (torch.arange(K, device=dev) % pad64(hd)) >= hd] = 0
            else:
                pad_rows = (torch.arange(N, device=dev) % pad64(hd)) >= hd
                w[pad_rows] = 0
                if b is not None:
                    b[pad_rows] = 0
    mk = (lambda *s: int_vec(g, *s)) if exact else (lambda *s: torch.randn(*s, generator=g, device=dev).half())
    if l.get("addend") == "scaled_residual":  # a ControlNet zero conv, at two conditioning scales
        for sc in (0.37, 2.0):
            run_scaled_residual(name, a, w, b, mk(M, N), sc, family=family)
        return
    a2 = None
    if l.get("k_split"):  # the dual-source shortcut: h and the skip connection, two buffers
        a, a2 = a[:, :l["k_split"]].contiguous(), a[:, l["k_split"]:].contiguous()
    lay = l.get("addend")
    addend = mk(M, N) if lay in ("residual", "in_place") else None
    run_linear(name, a, w, bias=b, addend=addend, a2=a2, geglu=geglu, in_place=lay == "in_place", family=family)


@pytest.mark.parametrize("launch", _production_cases())
def test_production_launch(launch):
    """Every GEMM / conv launch of the UNets, the VAE and the CLIP towers at production sizes and layouts: exact, and
    flat inputs (softmax rows for the VAE's P·V) under the bound."""
    run_production(launch, None)
    run_production(launch, "flat")


def test_vae_pv_softmax_families():
    """The VAE mid-block's P·V0 + b_v at K = 16384 (1024²), 15808 (1216x832), 9216 (768²) and 6144 (768x512): flat
    and peaked softmax rows of P against V0 at mean 10σ, the deepest accumulation of the project."""
    g = gen(77)
    for n, C in [(16384, 512), (15808, 512), (9216, 512), (6144, 512)]:
        w = (torch.randn(C, n, generator=g, device=dev) + 10).half()
        b = torch.randn(C, generator=g, device=dev).half()
        for peaked in (False, True):
            run_linear(f"vae P.V {n}x{C}x{n} {'peaked' if peaked else 'flat'} softmax", softmax_rows(g, n, n, peaked),
                       w, bias=b, family="softmax")


def check_launch_lists_against_profile(model, h, w, controlnet=False):
    """Build the native UNet (synthetic weights) at batch 2 on an h x w latent, profile one forward and compare its
    GEMM entries (kinds 0 / 1) with `unet_gemm_launches` and its attention entries (kind 2) with
    `production.unet_attn_launches`: the same names, kinds and algorithmic FLOPs. With `controlnet`, a ControlNet is
    attached: its `controlnet:` entries must equal `controlnet_body_launches` and the zero convs `zero_conv_launches`."""
    import production as P
    from cfgpp_b200 import config as C, controlnet as CN, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg = C.CONFIGS[model]()
    sd = Wt.synthetic_state_dict(cfg, seed=3, device=dev)
    net = NativeUNet(cfg, sd, dev)
    cn = None
    if controlnet:
        cn_cfg = CN.controlnet_config(cfg)
        cn = CN.NativeControlNet(cn_cfg, CN.synthetic_controlnet_state_dict(cn_cfg, seed=4, device=dev), dev)
    try:
        if cn is not None:
            net.attach_controlnet(cn)
        net.prepare(2, h, w)
        if cn is not None:
            net.set_control_image(torch.rand(2, 3, 8 * h, 8 * w, generator=torch.Generator().manual_seed(1)).to(dev))
        g = torch.Generator().manual_seed(0)
        ctx = torch.randn(4, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
        if cfg.addition_embed_type == "text_time":
            # original size, crop top-left, then the target size (base) or the aesthetic score (refiner)
            ids = [h * 8.0, w * 8, 0, 0, h * 8, w * 8][:cfg.num_time_ids]
            if cfg.num_time_ids == 5:
                ids[4] = 6.0
            net.set_prompt(ctx, torch.randn(4, cfg.pooled_dim, generator=g).half().to(dev),
                           torch.tensor([ids] * 4).to(dev))
        else:
            net.set_prompt(ctx)
        prof = net.profile_forward(torch.randn(2, 4, h, w, generator=g).to(dev), 500.0)
    finally:
        if cn is not None:
            cn.close()
        net.close()
        del sd
        torch.cuda.empty_cache()
    cnp = "controlnet:"
    if controlnet:
        got = sorted((n[len(cnp):], "conv" if k == 1 else "linear", f) for n, k, f, _ in prof
                     if k in (0, 1) and n.startswith(cnp))
        want = sorted((l["name"], l["kind"], l["flops"]) for l in controlnet_body_launches(cfg, h, w))
        assert len(got) == len(want), f"{len(got)} ControlNet GEMM launches reported, {len(want)} derived"
        for x, y in zip(got, want):
            assert x[:2] == y[:2] and abs(x[2] - y[2]) <= 1e-9 * y[2], f"ControlNet: reported {x}, derived {y}"
        zc = zero_conv_launches(cn_cfg, h, w)
        got = sorted((n, "conv" if k == 1 else "linear", f) for n, k, f, _ in prof
                     if k in (0, 1) and n.startswith("controlnet_"))
        want = sorted((l["name"], l["kind"], l["flops"]) for l in zc)
        assert len(got) == len(want), f"{len(got)} zero convs reported, {len(want)} derived"
        for x, y in zip(got, want):
            assert x[:2] == y[:2] and abs(x[2] - y[2]) <= 1e-9 * y[2], f"zero conv: reported {x}, derived {y}"
        prof = [e for e in prof if not e[0].startswith((cnp, "controlnet_"))]
    got = sorted((n, "conv" if k == 1 else "linear", f) for n, k, f, _ in prof if k in (0, 1))
    want = sorted((l["name"], l["kind"], l["flops"]) for l in unet_gemm_launches(cfg, h, w)
                  if l.get("plan") != "prompt")
    assert len(got) == len(want), f"{len(got)} GEMM launches reported, {len(want)} derived"
    for x, y in zip(got, want):
        assert x[:2] == y[:2] and abs(x[2] - y[2]) <= 1e-9 * y[2], f"reported {x}, derived {y}"
    got = sorted((n, f) for n, k, f, _ in prof if k == 2)
    want = sorted((l["name"], l["flops"]) for l in P.unet_attn_launches(cfg, h, w))
    assert len(got) == len(want), f"{len(got)} attention launches reported, {len(want)} derived"
    for x, y in zip(got, want):
        assert x[0] == y[0] and abs(x[1] - y[1]) <= 1e-9 * y[1], f"reported {x}, derived {y}"
    print(f"[gemm] {model} {8 * w}x{8 * h}{' + ControlNet' if controlnet else ''}: {len(prof)} profiled launches, "
          f"GEMM and attention lists match")


@pytest.mark.parametrize("model,hw", [("tiny_sdxl", 32), ("tiny_sd15", 32), ("sdxl", 128)])
def test_unet_launch_list_matches_profile(model, hw):
    """The derived UNet launch lists (GEMM: name, kind, algorithmic FLOPs; attention: name, FLOPs) equal the entries
    the native UNet's profile_forward reports for its body and tail plans, so the production lists cannot silently miss
    a launch."""
    check_launch_lists_against_profile(model, hw, hw)


@pytest.mark.parametrize("model,h,w", [("sd2", 96, 96), ("sd2", 96, 64), ("sdxl_refiner", 128, 128),
                                       ("sdxl_refiner", 152, 104)])
def test_unet_launch_list_matches_profile_rect(model, h, w):
    """The same cross-check for SD 2 at 768² and 768x512 and the SDXL refiner (5 time ids, 4 levels of 384..1536
    channels, about 4.5 GB of weights) at 1024² and 1216x832."""
    check_launch_lists_against_profile(model, h, w)


@pytest.mark.parametrize("model,hw", [("tiny_sd15", 32), ("tiny_sdxl", 32), ("sdxl", 128)])
def test_controlnet_launch_list_matches_profile(model, hw):
    """With a ControlNet attached: its body's `controlnet:` entries equal `controlnet_body_launches`, the zero convs
    equal `zero_conv_launches` (name, kind, FLOPs), and the UNet's own entries still equal its derived lists."""
    check_launch_lists_against_profile(model, hw, hw, controlnet=True)


@pytest.mark.parametrize("in_channels", P.T2I_IN_CHANNELS)
@pytest.mark.parametrize("model", list(P.T2I_ADAPTER_SIZES))
def test_t2i_adapter_launch_list_matches_plan_flops(model, in_channels):
    """The native T2I-Adapter (synthetic weights) at every production size and batch: the GEMM FLOPs its plan counts
    (`T2IAdapter::add_gemm`, GEMMs only) equal the sum over `t2i_adapter_gemm_launches`, so the derived list can
    neither miss nor invent a launch."""
    from cfgpp_b200 import config as C, t2i_adapter as T
    cfg = T.t2i_adapter_config(C.CONFIGS[model](), in_channels)
    ad = T.NativeT2IAdapter(cfg, T.synthetic_t2i_adapter_state_dict(cfg, seed=5, device=dev), dev)
    try:
        for h, w in P.T2I_ADAPTER_SIZES[model]:
            for B in P.T2I_ADAPTER_BATCHES:
                image = torch.rand(B, in_channels, 8 * h, 8 * w, generator=gen(B * h + w), device=dev)
                feats = ad.features(image)
                assert all(torch.isfinite(f).all() for f in feats)
                got = ad.stats["flops"]
                want = sum(l["flops"] for l in t2i_adapter_gemm_launches(cfg, 8 * h, 8 * w, B))
                print(f"[gemm] t2i {model} C{in_channels} {8 * w}x{8 * h} B{B}: plan {got:.6g} FLOPs, derived {want:.6g}")
                assert abs(got - want) <= 1e-9 * want, f"{model} {8 * w}x{8 * h} B{B}: plan {got}, derived {want}"
    finally:
        ad.close()


# ================================================================================================= coverage (last)

def test_zz_coverage():
    """Over the module: every tile width, both conv A-tile modes, natural and forced stream-K, tiles of >= 3 pieces,
    every addend mode (the ControlNet zero convs' scaled residual included) and the T2I-Adapter's convolutions on both
    A tiles at 1 and 8 images ran under the per-element gates. The 64-wide tile and the forced split are reached only
    by the launches that force them (the sweeps), so they are asserted when forced launches ran."""
    if SEEN["cases"] < 500:
        pytest.skip(f"only {SEEN['cases']} gated launches ran: coverage is asserted over the whole module")
    print(f"[gemm coverage] {SEEN['cases']} gated launches ({SEEN['forced']} forced): BN {sorted(SEEN['bn'])}, "
          f"A tile {sorted(SEEN['a_mode'])}, stream-K {sorted(str(s) for s in SEEN['streamk'])}, {SEEN['pieces3']} with "
          f">= 3 pieces per tile, addend {sorted(SEEN['addend'])}, T2I convs {sorted(SEEN['t2i_conv'])}")
    assert SEEN["bn"] >= {128, 160, 256}
    assert SEEN["a_mode"] >= {"linear", "tiled", "im2col"}
    assert SEEN["streamk"] >= {None, "natural"}
    assert SEEN["pieces3"] > 0
    assert SEEN["addend"] >= {"none", "residual", "temb_staged", "temb_rows", "scaled_residual"}
    assert SEEN["t2i_conv"] >= {(mode, B) for mode in ("tiled", "im2col") for B in (1, 8)}, SEEN["t2i_conv"]
    if SEEN["forced"]:
        assert 64 in SEEN["bn"]
        assert "forced" in SEEN["streamk"]
