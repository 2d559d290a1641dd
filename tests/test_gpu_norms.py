"""Kernel-level tests of GroupNorm(32)(+SiLU) (`gn_stats_kernel` + `gn_apply_kernel`) and LayerNorm (`layernorm_kernel`)
of `norm.cu`, through `cfgpp_op_groupnorm` / `cfgpp_op_layernorm`.

The reference is computed in fp64 on the GPU from the same fp16 inputs: per group (per row) μ, σ², rstd =
(σ² + eps)^-½, x̂ = (x − μ)·rstd, y = γ·x̂ + β, ref = y or silu(y). The gate is per element, |out − ref| ≤ E, with E
built from the kernel's rounding points (u = 2⁻²⁴):
  E_y   = |γ|·(|x̂|·ε_rstd + rstd·ε_mean) + 4u·(|γ·x̂| + |y|)
  E     = E_y                                                        without SiLU
        = 1.1·E_y + |ref|·((2 + 1.173·|y|)·2⁻²³ + 2⁻²² + u)           with SiLU
  gate  = E + ½ ulp_fp16(|ref| + E)                                  (the final rounding to fp16)
The affine step rounds x − μ, rstd·γ, the product and the + β (4u). silu is 1.1-Lipschitz, `__expf` is within
2 + 1.173·|y| ulp and `__fdividef` within 2 ulp.

ε_mean and ε_rstd are the first-order error bounds of a stable fp32 algorithm whose longest rounding chain is L steps,
taking 4 roundings per step (an add, a square or product, and Chan's correction term):
  ε_mean = 4·L·u·mean|x|,  ε_var = 4·L·u (relative),  ε_rstd = ½·ε_var + 2⁻²² (rsqrtf) + 2u (M2 / n, + eps).
GroupNorm's chain follows the launch geometry that `run_groupnorm` uses: a thread walks every pstep-th pixel of a
chunk of `gn_px_per_block(HW)` pixels (pstep = max(1, 256 / (C / 8))) in runs of m ≤ 32 pixels, merges its runs, the
pstep·cpg slots of a group are merged in turn, then every 8th chunk, then the 8 parts:
  L = m + runs per thread + pstep·cpg + ceil(nchunk / 8) + 8.
LayerNorm (one warp per row, two passes) chains 8·ceil(C / 256) values per lane and 5 shuffle steps:
  L = 8·ceil(C / 256) + 6, and ε_var also carries (ε_mean / σ)², the second pass's sum being taken about μ̂.
None of these depend on where the group's largest deviation lies. GroupNorm's statistics used to be sums shifted by a
single pivot sample (the group's first channel at pixel 0), whose error grows with the square of that sample's distance
from the mean; `test_groupnorm_outlier` puts an outlier of 30–1000σ there and at another pixel.

Every case asserts a finite output and prints its largest |err| / E and its rel-L2 (`pytest -s`). Inputs cover images
and groups with their own means (up to 100σ) and scales (2⁻⁶ to 2⁶), constant groups (exactly fp16(β)), variances
far below and near eps, sources at very different scales, HW from 1 pixel through chunk tails, C from 32 to 6144, and
every GroupNorm launch of the SDXL / SD v1.5 UNets and the VAE at production sizes. Bit-exact checks: dual source vs
the concatenated tensor, a batch vs its images, a permutation of whole groups, repeated launches, a LayerNorm row vs
the same row alone."""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
U = 2.0 ** -24
PIECE = 1 << 26  # fp64 elements of one slice of the reference


def ulp16(y):
    """Spacing of fp16 at |y| (fp64): 2^(e − 10) for |y| in [2^e, 2^(e+1)), 2^-24 in the subnormal range."""
    _, e = torch.frexp(y.abs())
    u = torch.ldexp(torch.ones_like(y), e - 11).clamp_min(2.0 ** -24)
    return torch.where(y == 0, torch.full_like(u, 2.0 ** -24), u)


def gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def cdiv(a, b):
    return -(-a // b)


def gn_chain(HW, C):
    """Longest rounding chain L of the GroupNorm statistics at this launch geometry (see the module docstring)."""
    ppb = max(4, cdiv(HW, 128))
    nchunk = cdiv(HW, ppb)
    pstep = max(1, 256 // (C // 8))
    per_thread = cdiv(min(ppb, HW), pstep)
    return min(32, per_thread) + cdiv(per_thread, 32) + pstep * (C // 32) + cdiv(nchunk, 8) + 8


class Gate:
    """Accumulates the worst |err| / E and the rel-L2 of one case over its slices."""
    def __init__(self, what):
        self.what = what
        self.worst = torch.zeros((), dtype=torch.float64, device=dev)
        self.err2, self.ref2 = self.worst.clone(), self.worst.clone()

    def add(self, o, ref, bound):
        assert torch.isfinite(o).all(), f"{self.what}: non-finite output"
        d = o - ref
        bound = bound + 0.5 * ulp16(ref.abs() + bound)
        self.worst = torch.maximum(self.worst, (d.abs() / bound).max())
        self.err2 += d.square().sum()
        self.ref2 += ref.square().sum()

    def done(self, tag):
        worst, rl = self.worst.item(), (self.err2 / self.ref2.clamp_min(1e-300)).sqrt().item()
        print(f"[{tag}] {self.what}: max |err|/E {worst:.3f}, rel-L2 {rl:.2e}")
        assert worst <= 1.0, f"{self.what}: error {worst:.3f}x the bound"
        return worst


def affine_bound(xh, rstd, e_mean, e_rstd, gam, y, ref, silu):
    e = gam.abs() * (xh.abs() * e_rstd + rstd * e_mean) + 4 * U * ((gam * xh).abs() + y.abs())
    if silu:
        e = 1.1 * e + ref.abs() * ((2 + 1.173 * y.abs()) * 2.0 ** -23 + 2.0 ** -22 + U)
    return e


def gn_check(what, x1, gamma, beta, eps, silu, x2=None):
    """Run GroupNorm on x1 [B, HW, C1] (+ x2 [B, HW, C2]) and gate every element against fp64. Returns the output."""
    from cfgpp_b200 import _native as nv
    out = nv.op_groupnorm(x1, gamma, beta, eps, silu, x2)
    B, HW, C1 = x1.shape
    C = C1 + (x2.shape[2] if x2 is not None else 0)
    cpg = C // 32
    L = gn_chain(HW, C)
    e_var = 4 * L * U
    e_rstd = 0.5 * e_var + 2.0 ** -22 + 2 * U
    gate = Gate(what)
    gs = max(1, min(32, PIECE // (HW * cpg)))
    for b in range(B):
        x = torch.cat([x1[b], x2[b]], 1) if x2 is not None else x1[b]
        for g0 in range(0, 32, gs):
            sl = slice(g0 * cpg, min(32, g0 + gs) * cpg)
            xg = x[:, sl].double().unflatten(1, (-1, cpg))  # [HW, groups, cpg]
            mu = xg.mean((0, 2), keepdim=True)
            var = (xg - mu).square().mean((0, 2), keepdim=True)
            rstd = (var + eps).rsqrt()
            e_mean = 4 * L * U * xg.abs().mean((0, 2), keepdim=True)
            xh = (xg - mu) * rstd
            del xg
            gam, bet = gamma[sl].double().view(1, -1, cpg), beta[sl].double().view(1, -1, cpg)
            y = xh * gam + bet
            ref = torch.nn.functional.silu(y) if silu else y
            bound = affine_bound(xh, rstd, e_mean, e_rstd, gam, y, ref, silu)
            del xh, y
            gate.add(out[b, :, sl].double().unflatten(1, (-1, cpg)), ref, bound)
    gate.done("groupnorm")
    return out


# ------------------------------------------------------------------------------------------------ GroupNorm inputs

def affine(g, C):
    """fp16 γ ~ N(1, 0.2²) and β ~ N(0, 0.2²)."""
    return ((torch.randn(C, generator=g, device=dev) * 0.2 + 1).half(),
            (torch.randn(C, generator=g, device=dev) * 0.2).half())


def gn_inputs(family, g, B, HW, C, *, mu_max=100.0):
    """fp16 x [B, HW, C] and γ, β [C] of one input family."""
    def rn(*s):
        return torch.randn(*s, generator=g, device=dev)

    def ru(*s, lo, hi):
        return torch.rand(*s, generator=g, device=dev) * (hi - lo) + lo

    x = rn(B, HW, C)
    if family == "homogeneous":
        x = x * 2 + 0.5
    elif family == "per_image":  # every image its own mean (up to 100 of its std) and scale 2^-6 .. 2^6
        s = torch.exp2(ru(B, 1, 1, lo=-6, hi=6))
        x = (x + ru(B, 1, 1, lo=-mu_max, hi=mu_max)) * s
    elif family == "per_group":  # every (image, group) its own mean (up to 100 of its std) and scale 2^-6 .. 2^6
        s = torch.exp2(ru(B, 1, 32, 1, lo=-6, hi=6))
        x = ((x.unflatten(2, (32, -1)) + ru(B, 1, 32, 1, lo=-mu_max, hi=mu_max)) * s).flatten(2)
    else:
        raise ValueError(family)
    return (x.half(), *affine(g, C))


def split(x, C1):
    return (x[..., :C1].contiguous(), x[..., C1:].contiguous()) if C1 < x.shape[2] else (x, None)


HW_SWEEP = (1, 2, 3, 4, 5, 7, 8, 127, 128, 129, 511, 512, 513, 1000)
C_SWEEP = (32, 64, 320, 640, 960, 1280, 2560, 6144)


@pytest.mark.parametrize("family", ["homogeneous", "per_image", "per_group"])
@pytest.mark.parametrize("C", C_SWEEP)
def test_groupnorm_sweep(C, family):
    """Every HW of the sweep (the 4-pixel minimum chunk, a partial last chunk, nchunk around multiples of 8) at
    B = 1, 3, 16; C from cpg = 1 to 6144, including C whose 256 / vpp leaves fewer than 256 threads (320, 960, 2560).
    Every other launch splits C into two sources at an 8-aligned channel inside a group."""
    g = gen(C * 7 + len(family))
    for B in (1, 3, 16):
        for i, HW in enumerate(HW_SWEEP):
            if B * HW * C > 1 << 26:
                continue
            x, gamma, beta = gn_inputs(family, g, B, HW, C)
            C1 = C if i % 2 == 0 or C < 64 else (C * 2 // 3) // 8 * 8
            x1, x2 = split(x, C1)
            gn_check(f"{family} B{B} HW{HW} C{C1}+{C - C1}", x1, gamma, beta, 1e-5, i % 3 != 2, x2)


@pytest.mark.parametrize("where", ["pivot", "other"])
@pytest.mark.parametrize("d", [30, 100, 300, 1000])
@pytest.mark.parametrize("B,HW,C1,C2", [(2, 16384, 320, 0), (2, 4096, 640, 320), (1, 65536, 128, 0), (3, 5, 64, 0)])
def test_groupnorm_outlier(B, HW, C1, C2, d, where):
    """N(0, 1) inputs with one sample d σ from the mean in every group of every image: at pixel 0 in the group's first
    channel (where a pivot-shifted sum would take its shift), or as a control at the last pixel in the group's middle
    channel. The bound does not depend on d."""
    C = C1 + C2
    cpg = C // 32
    g = gen(HW + C + d)
    x = torch.randn(B, HW, C, generator=g, device=dev)
    pix, ch = (0, 0) if where == "pivot" else (HW - 1, cpg // 2)
    sign = torch.randint(0, 2, (B, 32), generator=g, device=dev) * 2 - 1
    x[:, pix, ch::cpg] = d * sign
    gamma, beta = affine(g, C)
    x1, x2 = split(x.half(), C1)
    gn_check(f"outlier {d}σ at {where} B{B} HW{HW} C{C1}+{C2}", x1, gamma, beta, 1e-5, True, x2)


@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_constant_groups(silu):
    """Every other group is one constant (var = 0): x − μ is exactly 0 there, so the output is exactly fp16(β), or
    β through silu_f alone. The other groups are gated as usual."""
    for B, HW, C in [(2, 4096, 320), (3, 5, 64), (1, 1, 32), (2, 16384, 640)]:
        g = gen(HW + C + silu)
        cpg = C // 32
        x, gamma, beta = gn_inputs("per_group", g, B, HW, C, mu_max=10.0)
        const = torch.randn(B, 1, 32, 1, generator=g, device=dev).mul(30).half()
        xv = x.unflatten(2, (32, cpg))
        xv[:, :, ::2] = const[:, :, ::2]
        out = gn_check(f"constant groups silu={silu} B{B} HW{HW} C{C}", x, gamma, beta, 1e-5, silu)
        o = out.unflatten(2, (32, cpg))[:, :, ::2]
        bet = beta.view(32, cpg)[::2].expand_as(o)
        if silu:
            yb = bet.double()
            ref = torch.nn.functional.silu(yb)
            tol = 0.5 * ulp16(ref) + ref.abs() * ((2 + 1.173 * yb.abs()) * 2.0 ** -23 + 2.0 ** -22 + U)
            assert ((o.double() - ref).abs() <= tol).all(), "constant group: not silu(β)"
        else:
            assert torch.equal(o, bet), "constant group: not exactly β"


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("sigma", [1e-4, 3e-3])
def test_groupnorm_tiny_variance(eps, sigma):
    """0.5 + σ·N(0, 1) in fp16: a variance far below eps (σ = 1e-4, mostly one fp16 value) and near it (σ = 3e-3)."""
    g = gen(int(eps * 1e7) + int(sigma * 1e5))
    for B, HW, C1, C2 in [(2, 4096, 320, 0), (2, 1024, 640, 320), (3, 7, 64, 0)]:
        C = C1 + C2
        x = (0.5 + sigma * torch.randn(B, HW, C, generator=g, device=dev)).half()
        gamma, beta = affine(g, C)
        x1, x2 = split(x, C1)
        gn_check(f"tiny variance σ={sigma} eps={eps} B{B} HW{HW} C{C1}+{C2}", x1, gamma, beta, eps, True, x2)


def test_groupnorm_two_scales():
    """The two sources of a concat at scales 2^6 and 2^-6, so the groups that straddle C1 mix both."""
    g = gen(99)
    for B, HW, C1, C2 in [(2, 4096, 640, 320), (2, 1024, 1280, 640), (1, 129, 96, 32)]:
        x1 = (torch.randn(B, HW, C1, generator=g, device=dev) * 64 + 10).half()
        x2 = (torch.randn(B, HW, C2, generator=g, device=dev) / 64 - 0.01).half()
        C = C1 + C2
        gamma, beta = affine(g, C)
        gn_check(f"two scales B{B} HW{HW} C{C1}+{C2}", x1, gamma, beta, 1e-5, True, x2)


def test_groupnorm_channel_limits():
    """C % 32 != 0 raises, and so does C > 6144, whose shared-memory slots exceed the stats kernel's 48 KB."""
    from cfgpp_b200 import _native as nv
    for C1, C2 in [(40, 0), (320, 8), (6176, 0), (8192, 0), (4096, 4096)]:
        x1 = torch.zeros(1, 1, C1, dtype=torch.float16, device=dev)
        x2 = torch.zeros(1, 1, C2, dtype=torch.float16, device=dev) if C2 else None
        w = torch.zeros(C1 + C2, dtype=torch.float16, device=dev)
        with pytest.raises(nv.NativeError):
            nv.op_groupnorm(x1, w, w, 1e-5, True, x2)


# ------------------------------------------------------------------------------------------------ production shapes

def unet_gn_launches(cfg, h, w):
    """(C1, C2, HW, silu, eps) of every GroupNorm launch of a UNet on an h x w latent (diffusers' topology: resnets'
    norm1 / norm2, the transformers' norm, the up blocks' norm1 over concat(h, skip), conv_norm_out)."""
    ch, n, eps = cfg.block_out_channels, len(cfg.block_out_channels), cfg.norm_eps
    out = set()
    cur, skips = ch[0], [ch[0]]
    for i in range(n):
        HW = (h >> i) * (w >> i)
        for _ in range(cfg.layers_per_block):
            out |= {(cur, 0, HW, True, eps), (ch[i], 0, HW, True, eps)}
            cur = ch[i]
            if cfg.down_block_types[i].startswith("CrossAttn"):
                out.add((cur, 0, HW, False, 1e-6))
            skips.append(cur)
        if i < n - 1:
            skips.append(cur)
    HW = (h >> (n - 1)) * (w >> (n - 1))
    out |= {(cur, 0, HW, True, eps), (cur, 0, HW, False, 1e-6)}
    for j, i in enumerate(reversed(range(n))):
        HW = (h >> i) * (w >> i)
        for _ in range(cfg.layers_per_block + 1):
            out |= {(cur, skips.pop(), HW, True, eps), (ch[i], 0, HW, True, eps)}
            cur = ch[i]
            if cfg.up_block_types[j].startswith("CrossAttn"):
                out.add((cur, 0, HW, False, 1e-6))
    out.add((cur, 0, h * w, True, eps))
    assert not skips
    return sorted(out)


def vae_gn_launches(cfg, H, W):
    """(C, HW, silu) of every GroupNorm launch of the AutoencoderKL encoder and decoder on an H x W image."""
    ch, n, lpb = cfg.block_out_channels, len(cfg.block_out_channels), cfg.layers_per_block
    enc, dec = set(), set()
    cur = ch[0]
    for i in range(n):
        HW = (H >> i) * (W >> i)
        for _ in range(lpb):
            enc |= {(cur, HW, True), (ch[i], HW, True)}
            cur = ch[i]
    lo = (H >> (n - 1)) * (W >> (n - 1))
    enc |= {(cur, lo, True), (cur, lo, False)}  # mid resnets + attention, conv_norm_out
    cur = ch[-1]
    dec |= {(cur, lo, True), (cur, lo, False)}
    for i in reversed(range(n)):
        HW = (H >> i) * (W >> i)
        for _ in range(lpb + 1):
            dec |= {(cur, HW, True), (ch[i], HW, True)}
            cur = ch[i]
    dec.add((cur, H * W, True))
    return sorted(enc), sorted(dec)


def production_lists():
    """{(model, (h, w)): [(C1, C2, HW, silu, eps)]} of every UNet at every latent size of `production.py`, and
    {("vae", (H, W)): [(part, C, HW, silu)]} of the AutoencoderKL at every image size."""
    import production as P
    from cfgpp_b200 import config as C
    from cfgpp_b200.vae import VAEConfig
    out = {(m, (h, w)): unet_gn_launches(C.CONFIGS[m](), h, w) for m, h, w in P.unet_sizes()}
    for H, W in P.VAE_SIZES:
        enc, dec = vae_gn_launches(VAEConfig(), H, W)
        out[("vae", (H, W))] = [("decoder", *l) for l in dec] + [("encoder", *l) for l in enc]
    return out


def _unet_cases():
    """One case per launch over all UNets and sizes: SD 2-base repeats SD v1.5's list, which runs once."""
    seen, cases = set(), []
    for (m, (h, w)), launches in production_lists().items():
        for l in launches:
            if m != "vae" and l not in seen:
                seen.add(l)
                cases.append((m, h, w, *l))
    return cases


def test_unet_launch_list():
    """The derived SDXL list has the up blocks' straddling concat pairs (a group of 1920 = 1280 + 640 channels spans
    the boundary) and the transformers' eps-1e-6 norms."""
    from cfgpp_b200 import config as C
    sdxl = unet_gn_launches(C.CONFIGS["sdxl"](), 128, 128)
    assert (1280, 640, 32 * 32, True, 1e-5) in sdxl and (640, 320, 64 * 64, True, 1e-5) in sdxl
    assert any(c1 % ((c1 + c2) // 32) for c1, c2, *_ in sdxl if c2)
    assert (640, 0, 64 * 64, False, 1e-6) in sdxl and (320, 0, 128 * 128, True, 1e-5) in sdxl


@pytest.mark.parametrize("model,h,w,C1,C2,HW,silu,eps", _unet_cases())
def test_groupnorm_unet_launches(model, h, w, C1, C2, HW, silu, eps):
    """Every GroupNorm launch of every UNet at every latent size of `production.py`, at UNet batch 4, with per-image
    and per-group means and scales. The SDXL refiner brings 12..96 channels per group (384..3072 channels) and concat
    groups that straddle the source boundary (1536 + 768, 768 + 384); SD 2 at 768² puts 9216 pixels in a level."""
    g = gen(C1 * 3 + C2 + HW)
    x, gamma, beta = gn_inputs("per_group", g, 4, HW, C1 + C2, mu_max=30.0)
    x = (x.float() * torch.exp2(torch.rand(4, 1, 1, generator=g, device=dev) * 4 - 2)).half()
    x1, x2 = split(x, C1)
    gn_check(f"{model} {h}x{w} latent HW{HW} C{C1}+{C2} silu={silu} eps={eps}", x1, gamma, beta, eps, silu, x2)


def _vae_cases():
    """One case per (part, launch) over all VAE sizes."""
    seen, cases = set(), []
    for (m, (H, W)), launches in production_lists().items():
        for part, *l in launches:
            if m == "vae" and (part, *l) not in seen:
                seen.add((part, *l))
                cases.append((part, H, W, *l))
    return cases


@pytest.mark.parametrize("part,H,W,C,HW,silu", _vae_cases())
def test_groupnorm_vae_launches(part, H, W, C, HW, silu):
    """Every GroupNorm launch of the AutoencoderKL encoder and decoder at every image size of `production.py` (up to
    4 M elements per group at 1024²), per-group means and scales."""
    g = gen(C + HW)
    x, gamma, beta = gn_inputs("per_group", g, 1, HW, C, mu_max=30.0)
    gn_check(f"VAE {part} {H}x{W} HW{HW} C{C} silu={silu}", x, gamma, beta, 1e-6, silu)


# ------------------------------------------------------------------------------------------------ bit-exact checks

def test_groupnorm_bit_exact():
    """A dual-source launch equals the single-source launch on the concatenated tensor; a batch equals its images
    launched one by one; permuting whole groups (with γ, β) permutes the output; 10 launches are identical."""
    from cfgpp_b200 import _native as nv
    g = gen(3)
    for B, HW, C1, C2 in [(3, 4096, 640, 320), (2, 1000, 1280, 640), (4, 5, 96, 32)]:
        C = C1 + C2
        cpg = C // 32
        x, gamma, beta = gn_inputs("per_group", g, B, HW, C, mu_max=30.0)
        x1, x2 = split(x, C1)
        dual = nv.op_groupnorm(x1, gamma, beta, 1e-5, True, x2)
        assert torch.equal(dual, nv.op_groupnorm(x, gamma, beta, 1e-5, True)), "dual source != concat"
        for b in range(B):
            assert torch.equal(dual[b:b + 1], nv.op_groupnorm(x[b:b + 1].contiguous(), gamma, beta, 1e-5, True)), \
                f"image {b} differs from its own launch"
        perm = torch.randperm(32, generator=g, device=dev)
        cidx = (perm[:, None] * cpg + torch.arange(cpg, device=dev)).flatten()
        got = nv.op_groupnorm(x[..., cidx].contiguous(), gamma[cidx].contiguous(), beta[cidx].contiguous(), 1e-5, True)
        assert torch.equal(got, dual[..., cidx]), "group permutation does not permute the output"
        for _ in range(10):
            assert torch.equal(nv.op_groupnorm(x1, gamma, beta, 1e-5, True, x2), dual), "launches differ"


# ------------------------------------------------------------------------------------------------ moved rel-L2 cases

VAE_HW = 1024 * 1024  # the AutoencoderKL decoder's top level at 1024² (up to 4 M elements per group)


def check_groupnorm(B, HW, C1, C2, silu, eps, mu):
    """Sources at mean / std = mu (x1: std 2, x2: std 0.7)."""
    big = HW >= VAE_HW  # generated on the device: hundreds of millions of samples
    g = torch.Generator(device=dev if big else "cpu").manual_seed(C1 + C2 + mu)

    def src(*s, scale=1.0, shift=0.0):
        return (torch.randn(*s, generator=g, device=dev if big else "cpu") * scale + shift).half().to(dev)

    x1 = src(B, HW, C1, scale=2.0, shift=0.5 + 2.0 * mu)
    x2 = src(B, HW, C2, scale=0.7, shift=-0.3 - 0.7 * mu) if C2 else None
    Cc = C1 + C2
    gamma, beta = src(Cc, scale=0.2, shift=1.0), src(Cc, scale=0.2)
    gn_check(f"B{B} {HW}x{C1}+{C2} mu/sigma {mu}", x1, gamma, beta, eps, silu, x2)


@pytest.mark.parametrize("B,HW,C1,C2,silu,eps", [(2, 1024, 64, 0, True, 1e-5), (4, 16384, 320, 0, True, 1e-5),
                                                 (2, 4096, 640, 320, True, 1e-5), (2, 1024, 1280, 640, False, 1e-6)])
def test_groupnorm(B, HW, C1, C2, silu, eps):
    check_groupnorm(B, HW, C1, C2, silu, eps, 0)


@pytest.mark.parametrize("B,HW,C1,C2,silu,eps,mu", [
    (4, 16384, 320, 0, True, 1e-5, 10), (4, 16384, 320, 0, True, 1e-5, 30), (4, 16384, 320, 0, True, 1e-5, 100),
    (2, 4096, 640, 320, True, 1e-5, 10), (2, 4096, 640, 320, True, 1e-5, 30), (2, 4096, 640, 320, True, 1e-5, 100),
    (2, 1024, 1280, 640, False, 1e-6, 100),
    # the AutoencoderKL decoder's top level at 1024²: up to 4 M elements per group
    *[(1, VAE_HW, C, 0, True, 1e-6, mu) for C in (128, 256, 512) for mu in (0, 10, 30, 100)],
    (1, VAE_HW, 128, 128, True, 1e-6, 30)])
def test_groupnorm_mean_offset(B, HW, C1, C2, silu, eps, mu):
    """Inputs whose mean is mu times their std (E[x²] − E[x]² in fp32 would cancel away the variance), at UNet shapes
    and at the VAE decoder's top level, where fp32 sums run over millions of elements per group."""
    check_groupnorm(B, HW, C1, C2, silu, eps, mu)


# ------------------------------------------------------------------------------------------------ LayerNorm

def ln_check(what, x, gamma, beta, eps=1e-5):
    """Run LayerNorm on x [M, C] and gate every element against fp64. Returns the output."""
    from cfgpp_b200 import _native as nv
    out = nv.op_layernorm(x, gamma, beta, eps)
    M, C = x.shape
    L = 8 * cdiv(C, 256) + 6
    gate = Gate(what)
    rows = max(1, PIECE // C)
    for r0 in range(0, M, rows):
        xd = x[r0:r0 + rows].double()
        mu = xd.mean(1, keepdim=True)
        var = (xd - mu).square().mean(1, keepdim=True)
        rstd = (var + eps).rsqrt()
        e_mean = 4 * L * U * xd.abs().mean(1, keepdim=True)
        e_var = 4 * L * U + (e_mean * rstd).square()
        e_rstd = 0.5 * e_var + 2.0 ** -22 + 2 * U
        xh = (xd - mu) * rstd
        gam, bet = gamma.double(), beta.double()
        y = xh * gam + bet
        gate.add(out[r0:r0 + rows].double(), y, affine_bound(xh, rstd, e_mean, e_rstd, gam, y, y, False))
    gate.done("layernorm")
    return out


def ln_inputs(g, M, C, mu_max, const_every=0):
    """Rows with their own mean (up to mu_max of their std) and scale 2^-6 .. 2^3; every const_every-th row constant."""
    x = torch.randn(M, C, generator=g, device=dev)
    s = torch.exp2(torch.rand(M, 1, generator=g, device=dev) * 9 - 6)
    x = (x + (torch.rand(M, 1, generator=g, device=dev) * 2 - 1) * mu_max) * s
    if const_every:
        x[::const_every] = x[::const_every, :1]
    gamma = (torch.randn(C, generator=g, device=dev) * 0.2 + 1).half()
    beta = (torch.randn(C, generator=g, device=dev) * 0.2).half()
    return x.half(), gamma, beta


@pytest.mark.parametrize("mu_max", [0, 30, 1000])
@pytest.mark.parametrize("C", [8, 32, 320, 640, 768, 1280, 2048])
def test_layernorm_rows(C, mu_max):
    """Rows with their own mean (up to 1e3 σ) and scale at every M of the sweep; every 5th row constant, whose output
    is exactly fp16(β). C = 2048 fills all 8 vectors per lane."""
    g = gen(C + mu_max)
    for M in (1, 7, 9, 154, 4096):
        x, gamma, beta = ln_inputs(g, M, C, mu_max, const_every=5)
        out = ln_check(f"rows M{M} C{C} mu/sigma <= {mu_max}", x, gamma, beta)
        assert torch.equal(out[::5], beta.expand_as(out[::5])), "constant row: not exactly β"


def test_layernorm_bit_exact():
    """A row's output equals the same row normalised alone, and 10 launches are identical."""
    from cfgpp_b200 import _native as nv
    g = gen(17)
    for M, C in [(154, 2048), (4096, 640), (9, 8)]:
        x, gamma, beta = ln_inputs(g, M, C, 30)
        full = nv.op_layernorm(x, gamma, beta)
        for r in sorted({0, 1, M // 2, M - 1}):
            assert torch.equal(nv.op_layernorm(x[r:r + 1].contiguous(), gamma, beta), full[r:r + 1]), f"row {r}"
        for _ in range(10):
            assert torch.equal(nv.op_layernorm(x, gamma, beta), full)


def test_layernorm_channel_limits():
    """C = 12 (not a multiple of 8) and C = 2056 (over 8 vectors per lane) raise."""
    from cfgpp_b200 import _native as nv
    for C in (12, 2056):
        x = torch.zeros(2, C, dtype=torch.float16, device=dev)
        w = torch.zeros(C, dtype=torch.float16, device=dev)
        with pytest.raises(nv.NativeError):
            nv.op_layernorm(x, w, w)


def check_layernorm(M, Cc, mu):
    g = torch.Generator().manual_seed(M)

    def rnd(*s, scale=1.0, shift=0.0):
        return (torch.randn(*s, generator=g) * scale + shift).half().to(dev)

    x = rnd(M, Cc, scale=3.0, shift=1.0 + 3.0 * mu)
    gamma, beta = rnd(Cc, scale=0.2, shift=1.0), rnd(Cc, scale=0.2)
    ln_check(f"{M}x{Cc} mu/sigma {mu}", x, gamma, beta)


@pytest.mark.parametrize("M,Cc", [(4096, 1280), (16384, 640), (300, 128)])
def test_layernorm(M, Cc):
    check_layernorm(M, Cc, 0)


def test_layernorm_mean_offset():
    """Rows whose mean is 100 times their std (the kernel is two-pass: no cancellation in the variance)."""
    check_layernorm(4096, 1280, 100)


# ------------------------------------------------------------------------------------------------ LayerNorm launches

def layernorm_production_lists():
    """{key: [(case id, (M, C))]}: every LayerNorm launch of the text towers (layer_norm1 / 2 and final_layer_norm
    at M = 77·B), the vision towers (pre_layrnorm and the layers' norms at M = 257·B, post_layernorm over the B class
    rows) and an IP-Adapter's image_proj.norm (M = NB·tokens rows of width D at UNet batch NB = 4)."""
    import production as P
    from cfgpp_b200 import config as C
    from cfgpp_b200.text_encoder import CLIP_CONFIGS
    out = {}
    for tower, batches in P.TEXT_TOWERS.items():
        D = CLIP_CONFIGS[tower]().hidden_size
        for B in batches:
            out[(tower, B)] = [(f"{tower}-B{B}-layer_norm", (P.N_CTX * B, D))]
    for tower, batches in P.VISION_TOWERS.items():
        v = P.vision_config(tower)
        for B in batches:
            out[(tower, B)] = [(f"{tower}-B{B}-layer_norm", (v.num_positions * B, v.hidden_size)),
                               (f"{tower}-B{B}-post_layernorm", (B, v.hidden_size))]
    for m, E in P.IP_ADAPTERS:
        D = C.CONFIGS[m]().cross_attention_dim
        out[("ip_adapter", m, E)] = [(f"ip-{m}-image_proj.norm", (4 * P.IP_TOKENS, D))]
    return out


def _layernorm_cases():
    seen, cases = set(), []
    for launches in layernorm_production_lists().values():
        for cid, s in launches:
            if s not in seen:
                seen.add(s)
                cases.append(pytest.param(*s, id=cid))
    return cases


@pytest.mark.parametrize("M,C", _layernorm_cases())
def test_layernorm_production_launches(M, C):
    """Every LayerNorm launch of the text and vision towers and the IP-Adapter projection, per element against fp64:
    rows with their own mean (up to 30σ) and scale; from 14 rows on every 7th row constant (exactly fp16(β))."""
    g = gen(M * 7 + C)
    every = 7 if M >= 14 else 0
    x, gamma, beta = ln_inputs(g, M, C, 30, const_every=every)
    out = ln_check(f"production M{M} C{C}", x, gamma, beta)
    if every:
        assert torch.equal(out[::7], beta.expand_as(out[::7])), "constant row: not exactly β"
