"""Kernel-level tests of the flash-attention kernel `attn_kernel<HD>` (`attention.cu`) through `cfgpp_op_attention`.

The reference is computed in fp64 on the GPU from the same fp16 inputs, over the real head_dim columns only:
s = q·k / sqrt(head_dim), p = softmax(s), ref = p @ v. The gate is per element, |out − ref| ≤ E, where E is the
error bound of the kernel's rounding points (`_reference` derives it). Every case prints the largest |err| / E and the
rel-L2 against the fp64 reference (`pytest -s`), asserts a finite output and exact +0 in the padding columns of padded
heads. The inputs cover flat and peaked softmaxes, a running max that rises in every KV tile or sits in tile 0, a hot
key in the last partial tile, P values that underflow fp16, large and offset values and extreme logits, at every tile
boundary of Nq / Nkv and at the UNets' production shapes and layouts.

Each CTA owns one (64-row query tile, head, batch) and walks the KV tiles in a fixed order, so some results are
determined bit for bit: known answers (identical keys; one key ≥ 40 nats above the rest), the fused QKV / KV layouts
against contiguous copies, batch independence, head permutation, row truncation and determinism."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

HEAD_DIMS = (64, 40, 80, 160)  # SDXL; SD v1.5 (padded to 64 / 128 / 192 columns)
NQ_SWEEP = (1, 63, 64, 65, 130)
# the mask tests the two columns of a lane's pair separately, so a last tile with an even count of valid columns
# (2, 36) is the one where an off-by-one in the even column's test lets a padding key in
NKV_SWEEP = (1, 2, 63, 64, 65, 100, 127, 128, 129, 191, 192, 193)
FAMILIES = ("flat", "peaked", "rising", "falling", "hot_last", "hot_tile", "huge_range", "large_v", "offset_v",
            "extreme")
SCORE_CHUNK = 1 << 24  # fp64 elements of one [heads, Nq, Nkv] block of the reference
PIECE = 1 << 25  # fp64 elements of one [rows, Nkv, head_dim] piece of the bound's last term


def padded(hd):
    return (hd + 63) // 64 * 64


def bits(t):
    return t.view(torch.int16)


def ulp16(y):
    """Spacing of fp16 at |y| (fp64): 2^(e − 10) for |y| in [2^e, 2^(e+1)), 2^-24 in the subnormal range."""
    _, e = torch.frexp(y.abs())
    u = torch.ldexp(torch.ones_like(y), e - 11).clamp_min(2.0 ** -24)
    return torch.where(y == 0, torch.full_like(u, 2.0 ** -24), u)


def heads(t, hdp):
    """[B, N, H, hd] -> [B, N, H·hdp] fp16, every head zero-padded to hdp columns (the UNets' packed head layout)."""
    B, N, H, hd = t.shape
    out = torch.zeros(B, N, H, hdp, dtype=torch.float16, device=dev)
    out[..., :hd] = t
    return out.flatten(2)


def fused(*ts):
    """Column slices of one [B, N, len(ts)·C] buffer, as the fused QKV (self) and KV (cross) projections write them."""
    buf = torch.cat(ts, 2)
    C = ts[0].shape[2]
    return [buf[:, :, i * C:(i + 1) * C] for i in range(len(ts))]


def _reference(q, k, v, hdp):
    """fp64 attention of one block of heads, q [G, Nq, hd], k / v [G, Nkv, hd], and the per-element bound E of the
    kernel's error. The kernel rounds at these points, and each gets a term of E:
      ½ ulp_fp16(ref)                       the output's final rounding to fp16;
      (2^-11 + (Nkv + 8)·2^-24)·Σ_j p_j|v_j|  P rounded to fp16 before PV (relative 2^-11; l sums the unrounded p, so
                                            only PV sees it), ex2.approx (≤ 2^-22 relative, in PV and l alike) and the
                                            fp32 sums of l and O (one rounding per added term, at most Nkv of them);
      2^-25·Σ_j |v_j| / L                   P in fp16's subnormal range: an absolute error of up to half the spacing
                                            2^-24, in units of the tile's running max, which is at most the final max;
                                            L = Σ_j exp(s_j − max s);
      2·Σ_j p_j·δ_j·|v_j − ref|             an error δ_j in the exponent of key j moves the output by
                                            p_j·δ_j·(v_j − ref) to first order (l and PV move together);
                                            the 2 covers the second order.
    δ_j = (hdp + 2)·2^-24·scale·Σ_d|q_d k_jd| is the fp32 dot product over the padded head, and 2^-22·(|s_j| + max|s|)
    covers the separate fp32 roundings of s·log2e and m·log2e before they are subtracted, and of scale·log2e itself.
    O and l are rescaled by the same alpha each tile, so alpha's own ex2 error cancels; its argument's rounding is a
    shift of the exponent of every earlier key, inside the same δ term."""
    G, Nq, hd = q.shape
    Nkv = k.shape[1]
    scale = hd ** -0.5
    s = (q @ k.mT).mul_(scale)
    p = torch.exp(s - s.amax(-1, keepdim=True))
    L = p.sum(-1, keepdim=True)
    p.div_(L)
    ref = p @ v
    av = v.abs()
    w = (q.abs() @ k.abs().mT).mul_((hdp + 2) * 2.0 ** -24 * scale)
    s.abs_()
    w.add_((s + s.amax(-1, keepdim=True)).mul_(2.0 ** -22)).mul_(p)  # p_j δ_j
    del s
    bound = (0.5 * ulp16(ref) + (2.0 ** -11 + (Nkv + 8) * 2.0 ** -24) * (p @ av)
             + 2.0 ** -25 * av.sum(1, keepdim=True) / L)
    rows = max(1, PIECE // (Nkv * hd))
    for g in range(G):
        for i in range(0, Nq, rows):
            r = slice(i, i + rows)
            bound[g, r] += 2 * (v[g, None] - ref[g, r, None]).abs_().mul_(w[g, r, :, None]).sum(1)
    return ref, bound


def check(what, q, k, v, H, hd):
    """Run the kernel on q [B, Nq, H·hdp], k / v [B, Nkv, H·hdp] (views with a row stride allowed) and gate every
    element against the fp64 reference. Returns the output."""
    from cfgpp_b200 import _native as nv
    out = nv.op_attention(q, k, v, H, head_dim=hd)
    B, Nq, C = q.shape
    Nkv, hdp = k.shape[1], C // H
    o = out.unflatten(2, (H, hdp))
    assert torch.isfinite(o).all(), f"{what}: non-finite output"
    if hdp > hd:
        assert (bits(o[..., hd:]) == 0).all(), f"{what}: padding columns are not +0"
    qh, kh, vh = (t.unflatten(2, (H, hdp))[..., :hd] for t in (q, k, v))
    G = max(1, min(H, SCORE_CHUNK // (Nq * Nkv)))
    worst = torch.zeros((), dtype=torch.float64, device=dev)
    err2, ref2 = worst.clone(), worst.clone()
    for b in range(B):
        for h0 in range(0, H, G):
            hs = slice(h0, min(H, h0 + G))
            ref, bound = _reference(*(t[b, :, hs].transpose(0, 1).double() for t in (qh, kh, vh)), hdp)
            d = o[b, :, hs, :hd].transpose(0, 1).double() - ref
            worst = torch.maximum(worst, (d.abs() / bound).max())
            err2 += d.square().sum()
            ref2 += ref.square().sum()
    worst, rl = worst.item(), (err2 / ref2.clamp_min(1e-300)).sqrt().item()
    print(f"[attention] {what}: max |err|/E {worst:.3f}, rel-L2 {rl:.2e}")
    assert worst <= 1.0, f"{what}: error {worst:.3f}x the bound"
    return out


def family(name, g, B, Nq, Nkv, H, hd):
    """Inputs of one family: q [B, Nq, H, hd], k / v [B, Nkv, H, hd], fp32 on the device (rounded to fp16 by the
    caller). Scaled logits s = q·k / sqrt(hd) have a std of about σ_q σ_k."""
    def rn(*s):
        return torch.randn(*s, generator=g, device=dev)

    q, k, v = rn(B, Nq, H, hd), rn(B, Nkv, H, hd), rn(B, Nkv, H, hd)
    u = torch.randint(0, 2, (H, hd), generator=g, device=dev).float() * 2 - 1  # a shared ±1 direction, |u|² = hd
    if name == "flat":  # the softmax is nearly flat: logit std ≈ 1.4
        return 1.2 * q, 1.2 * k, 1.2 * v
    if name == "peaked":  # logit std ≈ 9, as in trained UNets' attention
        return 3 * q, 3 * k, v
    if name == "huge_range":  # logit std ≈ 20: most keys are over 40 nats below the max, their fp16 P values are 0
        return 4.5 * q, 4.5 * k, v
    if name in ("rising", "falling"):  # logits ≈ t_j·sqrt(hd) ± 0.7: the running max rises in every KV tile, or
        t = torch.linspace(0, 1, Nkv, device=dev)  # sits in tile 0 and alpha stays 1
        if name == "falling":
            t = t.flip(0)
        return 0.5 * q + u, 0.5 * k + t[:, None, None] * u, v
    if name in ("hot_last", "hot_tile"):  # one key ≈ 12 nats above the rest (std ≈ 1.9), at column Nkv − 1 or at the
        col = Nkv - 1 if name == "hot_last" else (Nkv - 1) // 64 * 64  # first column of the last (partial) tile
        k = 1.2 * k
        k[:, col] = u * (12 / math.sqrt(hd))
        return 1.2 * q + u, k, v
    if name == "large_v":
        return 1.2 * q, 1.2 * k, 1e3 * v
    if name == "offset_v":  # v's mean is 100 times its std
        return 1.2 * q, 1.2 * k, v + 100
    if name == "extreme":  # |q|, |k| entries up to 60: logits in the thousands
        return ((torch.rand(B, Nq, H, hd, generator=g, device=dev) * 2 - 1) * 60,
                (torch.rand(B, Nkv, H, hd, generator=g, device=dev) * 2 - 1) * 60, v)
    raise ValueError(name)


def gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


@pytest.mark.parametrize("hd", HEAD_DIMS)
@pytest.mark.parametrize("name", FAMILIES)
def test_tile_boundary_sweep(name, hd):
    """Every family at every Nq / Nkv around the 64-row tiles (a partial last query tile, a partial last KV tile with
    1, 2, 36 or 63 valid columns, one to four KV tiles), B = 1 and 3, two heads; k / v are slices of one fused KV
    buffer."""
    H, hdp = 2, padded(hd)
    g = gen(FAMILIES.index(name) * 1000 + hd)
    for B in (1, 3):
        for Nq in NQ_SWEEP:
            for Nkv in NKV_SWEEP:
                q, k, v = family(name, g, B, Nq, Nkv, H, hd)
                k, v = fused(heads(k, hdp), heads(v, hdp))
                check(f"{name} hd{hd} B{B} {Nq}x{Nkv}", heads(q, hdp), k, v, H, hd)


def production_lists():
    """{(model, (h, w)): [(case id, (heads, Nq, Nkv, head_dim))]}: the distinct attention shapes of every UNet at every
    latent size of `production.py` (self-attention and cross-attention per attention level and the mid block)."""
    import production as P
    from cfgpp_b200 import config as C
    out = {}
    for m, h, w in P.unet_sizes():
        shapes = []
        for l in P.unet_attn_launches(C.CONFIGS[m](), h, w):
            s = (l["heads"], l["Nq"], l["Nkv"], l["hd"])
            if s not in shapes:
                shapes.append(s)
        out[(m, (h, w))] = [(f"{P.size_tag(m, h, w)}-{'self' if s[1] == s[2] else 'cross'}-H{s[0]}-{s[1]}x{s[2]}"
                             f"-hd{s[3]}", s) for s in shapes]
    return out


def _production_cases():
    """One case per shape over all models and sizes, under the id of the first (model, size) that has it."""
    seen, cases = set(), []
    for shapes in production_lists().values():
        for cid, s in shapes:
            if s not in seen:
                seen.add(s)
                cases.append(pytest.param(*s, id=cid))
    return cases


@pytest.mark.parametrize("name", ["flat", "peaked"])
@pytest.mark.parametrize("H,Nq,Nkv,hd", _production_cases())
@pytest.mark.parametrize("NB", [4, 16])
def test_production_shapes(NB, H, Nq, Nkv, hd, name):
    """Every attention shape of the UNets' transformer blocks at every production size (`production.py`: SDXL and
    the refiner at 1024² and 1216x832, whose 76x52 = 3952-token level ends in a 48-column KV tile after 61 full ones;
    the refiner at 1344x768; SD 2 at 768² (9216 tokens) and 768x512; SD v1.5 and SD 2-base at 512²), at UNet batch
    NB = 4 / 16 (B = 2 / 8 images with CFG), in the layouts the UNet launches: self-attention reads q / k / v as column
    slices of the fused [NB, N, 3·H·hdp] QKV buffer, cross-attention reads K / V as slices of the prompt's
    [NB, 77, 2·H·hdp] KV buffer and q from its own [NB, N, H·hdp] buffer."""
    hdp = padded(hd)
    g = gen(NB * 100003 + Nq * 1009 + Nkv * 7 + hd + (name == "peaked"))
    q, k, v = (heads(t, hdp) for t in family(name, g, NB, Nq, Nkv, H, hd))
    if Nq == Nkv:
        q, k, v = fused(q, k, v)
    else:
        k, v = fused(k, v)
    check(f"{name} NB{NB} H{H} {Nq}x{Nkv} hd{hd}", q, k, v, H, hd)


def vision_production_lists():
    """{(tower, B): [(case id, (B, heads, T, head_dim))]}: the non-causal self-attention of every CLIP vision tower of
    `production.VISION_TOWERS` (T = (image_size / patch_size)² + 1 tokens) at each image batch."""
    import production as P
    out = {}
    for tower, batches in P.VISION_TOWERS.items():
        v = P.vision_config(tower)
        H, T = v.num_attention_heads, v.num_positions
        for B in batches:
            s = (B, H, T, v.hidden_size // H)
            out[(tower, B)] = [(f"{tower}-B{B}-H{H}-{T}x{T}-hd{s[3]}", s)]
    return out


def _vision_cases():
    seen, cases = set(), []
    for shapes in vision_production_lists().values():
        for cid, s in shapes:
            if s not in seen:
                seen.add(s)
                cases.append(pytest.param(*s, id=cid))
    return cases


@pytest.mark.parametrize("name", ["flat", "peaked"])
@pytest.mark.parametrize("B,H,T,hd", _vision_cases())
def test_vision_tower_shapes(B, H, T, hd, name):
    """The CLIP vision towers' self-attention (ViT-H: heads of 80, ViT-bigG: heads of 104, both padded to 128 columns)
    over 257 tokens (four full KV tiles and one of a single key), reading q / k / v as column slices of the fused
    [B·257, 3·Cp] buffer the qkv GEMM writes."""
    hdp = padded(hd)
    g = gen(B * 100003 + T * 1009 + hd + (name == "peaked"))
    q, k, v = fused(*(heads(t, hdp) for t in family(name, g, B, T, T, H, hd)))
    check(f"vision {name} B{B} H{H} {T}x{T} hd{hd}", q, k, v, H, hd)


# ---- cases of the earlier rel-L2 tests, under the per-element gate -----------------------------------------------

def rnd(g, *s, scale=1.0):
    return (torch.randn(*s, generator=g) * scale).half().to(dev)


@pytest.mark.parametrize("B,H,Nq,Nkv", [(1, 1, 128, 128), (1, 4, 64, 64), (2, 5, 1024, 1024), (1, 10, 4096, 4096),
                                        (4, 20, 1024, 77), (1, 2, 200, 333), (1, 1, 1, 1),
                                        # one KV tile (cross-attention): partial KV tiles, a partial last query tile
                                        (4, 10, 4096, 77), (1, 5, 1024, 128), (2, 3, 520, 100), (1, 2, 256, 5),
                                        # the bench shape, ragged Nq / Nkv, many heads
                                        (4, 20, 1024, 1024), (3, 13, 1100, 1000), (1, 37, 1024, 640), (2, 31, 700, 333)])
def test_attention(B, H, Nq, Nkv):
    """Head dim 64, flat inputs; q / k / v slices of one fused buffer for self-attention, k / v for cross-attention."""
    g = torch.Generator().manual_seed(Nq + Nkv)
    Cc = H * 64
    if Nq == Nkv:
        qkv = rnd(g, B, Nq, 3 * Cc, scale=1.2)
        q, k, v = qkv[:, :, :Cc], qkv[:, :, Cc:2 * Cc], qkv[:, :, 2 * Cc:]
    else:
        q, kv = rnd(g, B, Nq, Cc, scale=1.2), rnd(g, B, Nkv, 2 * Cc, scale=1.2)
        k, v = kv[:, :, :Cc], kv[:, :, Cc:]
    check(f"B{B} H{H} {Nq}x{Nkv}", q, k, v, H, 64)


@pytest.mark.parametrize("B,H,Nq,Nkv,hd", [(2, 8, 1024, 1024, 80), (1, 8, 4096, 4096, 40), (2, 8, 256, 256, 160),
                                           (2, 8, 64, 77, 160), (1, 3, 300, 77, 40), (2, 8, 1024, 77, 80),
                                           (2, 8, 256, 77, 160), (1, 4, 4096, 77, 40), (1, 2, 640, 120, 160),
                                           (2, 8, 4096, 4096, 40)])
def test_attention_padded_heads(B, H, Nq, Nkv, hd):
    """SD v1.5 head dims (40 / 80 / 160), zero-padded to a multiple of 64 columns, as separate contiguous tensors."""
    g = torch.Generator().manual_seed(hd + Nq)
    P = padded(hd)

    def pad(n):
        t = torch.zeros(B, n, H, P)
        t[..., :hd] = torch.randn(B, n, H, hd, generator=g) * 1.1
        return t.reshape(B, n, H * P).half().to(dev)

    check(f"hd{hd} B{B} H{H} {Nq}x{Nkv}", pad(Nq), pad(Nkv), pad(Nkv), H, hd)


# ---- bit-exact properties ----------------------------------------------------------------------------------------

def attention(q, k, v, H, hd):
    from cfgpp_b200 import _native as nv
    return nv.op_attention(q, k, v, H, head_dim=hd)


@pytest.mark.parametrize("hd", HEAD_DIMS + (104,))
def test_known_answer_uniform_keys(hd):
    """Every key row is the same and every value row is the same row v0: all scores of a query row are equal, every p
    is 1 and the output is v0 bit for bit. The logits are small (std ≈ 0.3) and of both signs, so one padding key of
    the partial last tile (score 0, value 0) let through the mask would move the output by far more than an ulp."""
    B, H, hdp = 2, 2, padded(hd)
    g = gen(hd)
    for Nq in NQ_SWEEP:
        for Nkv in NKV_SWEEP:
            q = torch.randn(B, Nq, H, hd, generator=g, device=dev)
            k0 = 0.3 * torch.randn(B, 1, H, hd, generator=g, device=dev)
            v0 = heads(torch.randn(B, 1, H, hd, generator=g, device=dev), hdp)
            k, v = fused(heads(k0.expand(B, Nkv, H, hd), hdp), v0.expand(B, Nkv, H * hdp))
            out = attention(heads(q, hdp), k, v, H, hd)
            assert torch.equal(out, v0.expand(B, Nq, H * hdp)), f"hd{hd} {Nq}x{Nkv}: output != v0"


@pytest.mark.parametrize("hd", HEAD_DIMS + (104,))
def test_known_answer_one_hot(hd):
    """One key ≈ 70 nats above every other (≥ 47 above the 'warm' keys, ≈ 68 above the rest): every other p is below
    e^-40 and rounds to 0 in fp16, so the output is that key's value row bit for bit. The hot key sits at column 0, in
    a middle tile, at the first and at the last valid column of the last partial tile; in the last case, warm keys
    (≈ 20 nats) in earlier tiles make the running max jump, and alpha ≈ e^-50 must wipe what those tiles added."""
    B, H, Nq, hdp = 2, 2, 130, padded(hd)
    g = gen(hd + 7)
    u = torch.ones(H, hd, device=dev)
    for Nkv in (77, 150, 193):
        last = (Nkv - 1) // 64 * 64
        cases = [(c, ()) for c in sorted({0, last, Nkv - 1} | ({64 + 29} if Nkv > 128 else set()))]
        cases.append((Nkv - 1, (3, 64 + 5) if Nkv > 128 else (3,)))
        for hot, warm in cases:
            q = u + 0.05 * torch.randn(B, Nq, H, hd, generator=g, device=dev)
            k = 0.5 * torch.randn(B, Nkv, H, hd, generator=g, device=dev)
            k[:, hot] = u * (70 / math.sqrt(hd))
            for c in warm:
                k[:, c] = u * (20 / math.sqrt(hd))
            v = heads(torch.randn(B, Nkv, H, hd, generator=g, device=dev), hdp)
            k, v = fused(heads(k, hdp), v)
            out = attention(heads(q, hdp), k, v, H, hd)
            want = v[:, hot:hot + 1].expand(B, Nq, H * hdp)
            assert torch.equal(out, want), f"hd{hd} Nkv {Nkv}: hot key at {hot} (warm {warm}): output != its value row"


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_layout_invariance(hd):
    """q / k / v as column slices of one fused [B, N, 3·H·hdp] buffer (self-attention), and k / v as slices of one
    [B, Nkv, 2·H·hdp] buffer (cross-attention), give the same output as contiguous copies."""
    B, H, N, Nkv, hdp = 2, 3, 300, 77, padded(hd)
    g = gen(hd + 11)
    q, k, v = (heads(t, hdp) for t in family("peaked", g, B, N, N, H, hd))
    fq, fk, fv = fused(q, k, v)
    assert torch.equal(check(f"fused qkv hd{hd} B{B} H{H} {N}x{N}", fq, fk, fv, H, hd), attention(q, k, v, H, hd))
    q, k, v = (heads(t, hdp) for t in family("peaked", g, B, N, Nkv, H, hd))
    fk, fv = fused(k, v)
    assert torch.equal(check(f"fused kv hd{hd} B{B} H{H} {N}x{Nkv}", q, fk, fv, H, hd), attention(q, k, v, H, hd))


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_batch_head_and_row_independence(hd):
    """A batch-3 launch equals three batch-1 launches on its slices; permuting the head blocks of q / k / v permutes
    the output's head blocks the same way; rows [0, n) of a launch on the first n query rows (n not a multiple of 64)
    equal the same rows of the full launch."""
    B, H, Nq, Nkv, hdp = 3, 5, 300, 200, padded(hd)
    g = gen(hd + 13)
    q, k, v = (heads(t, hdp) for t in family("peaked", g, B, Nq, Nkv, H, hd))
    full = attention(q, k, v, H, hd)
    for b in range(B):
        assert torch.equal(attention(q[b:b + 1], k[b:b + 1], v[b:b + 1], H, hd), full[b:b + 1]), f"batch {b}"
    perm = [3, 0, 4, 1, 2]

    def permute(t):
        return t.unflatten(2, (H, hdp))[:, :, perm].flatten(2)

    assert torch.equal(attention(permute(q), permute(k), permute(v), H, hd), permute(full)), "head permutation"
    for n in (1, 100, 257):
        assert torch.equal(attention(q[:, :n].contiguous(), k, v, H, hd), full[:, :n]), f"first {n} rows"


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_determinism(hd):
    """Ten back-to-back launches give identical outputs."""
    B, H, N, hdp = 2, 8, 1024, padded(hd)
    q, k, v = fused(*(heads(t, hdp) for t in family("peaked", gen(hd + 17), B, N, N, H, hd)))
    outs = [attention(q, k, v, H, hd) for _ in range(10)]
    for i, o in enumerate(outs[1:], 1):
        assert torch.equal(o, outs[0]), f"launch {i} differs from launch 0"
