"""Kernel-level tests of the small hand-written kernels every image passes through, through their C-ABI entry points:
the UNet's timestep embedding, tiny-M linear, row copy, conv_in, conv_out fused with the CFG++ step and nearest-2x
upsample (`elementwise.cu`); the AutoencoderKL's latent preparation, row softmax, RGB conv_out, image pad and
encoder moments / sample (`vae_kernels.cu`); the CLIP towers' embedding, causal attention, MLP activation and pooled-row
gather (`text_kernels.cu`).

Every reference takes the same fp16 inputs, accumulates in fp64 and rounds to fp16 where the reference model's fp16
autocast graph does. Where the arithmetic is determined (copies, gathers, one fp16 add, the step applied to the eps the
same launch wrote, the activations against torch on the same GPU) the test asserts bit-equality; elsewhere the gates
are ≈5x the error observed on an H100 and every test prints what it measured (`pytest -s`)."""
import math

import pytest
import torch
import torch.nn.functional as F

from cfgpp_b200.config import sdxl_refiner_config
from helpers import coef_variants, rel_l2

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

TOL_GEMM = 2e-4  # fp32 accumulation vs fp64, both rounded once to fp16: only last-bit flips remain


def gate(what, got, ref, tol):
    e = rel_l2(got, ref)
    print(f"[small kernels] {what}: rel-L2 {e:.3e} (gate {tol:.1e})")
    assert e < tol, f"{what}: rel-L2 {e:.3e} >= {tol:.1e}"
    return e


def rnd(g, *s, scale=1.0, shift=0.0):
    return (torch.randn(*s, generator=g) * scale + shift).half().to(dev)


def ulp16(y, normal_only=False):
    """Spacing of fp16 at |y| (fp64 tensor): 2^(e - 10) for |y| in [2^e, 2^(e+1)); 2^-24 below the normal range unless
    normal_only, which keeps the normal-range formula (so that a gate of max(ulp16, 2^-25) is the subnormal
    half-spacing there)."""
    m, e = torch.frexp(y.double().abs())
    u = torch.ldexp(torch.ones_like(m), (e - 11).to(torch.int32))
    u = torch.where(y == 0, torch.full_like(u, 2.0 ** -25 if normal_only else 2.0 ** -24), u)
    return u if normal_only else u.clamp_min(2.0 ** -24)


def border_mask(H, W):
    m = torch.zeros(H, W, dtype=torch.bool, device=dev)
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = True
    return m


def bits(t):
    return t.contiguous().view(torch.int16)


# ---- timestep embedding -----------------------------------------------------------------------------------------

def _sincos_ref(vals, dim):
    """diffusers get_timestep_embedding (flip_sin_to_cos, shift 0) as torch runs it on the GPU: fp32 frequency (the
    division of the exponent by half_dim, a Python scalar, is a multiplication by its fp32 reciprocal there) and fp32
    argument, then exact (fp64) cos | sin. Returns (ref [n, dim] fp64, |argument| [n, dim/2] fp64)."""
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(0, half, dtype=torch.float32, device=dev) / half
    arg = vals.float()[:, None] * torch.exp(exponent)[None, :]
    a = arg.double()
    return torch.cat([torch.cos(a), torch.sin(a)], 1), a.abs()


def _check_sincos(what, got, vals, dim):
    ref, a = _sincos_ref(vals, dim)
    # half an fp16 ulp for the output rounding, the fp32 argument's own rounding (a frequency 1 ulp off moves the
    # argument by |t f_k| 2^-23) and 4 fp32 ulp for cosf / sinf
    bound = 0.5 * ulp16(ref) + torch.cat([a, a], 1) * 2.0 ** -23 + ref.abs() * 2.0 ** -21
    err = (got.double() - ref).abs()
    worst = (err / bound).max().item()
    print(f"[small kernels] {what}: max |err| {err.max().item():.3e}, max err/bound {worst:.3f}")
    assert worst <= 1.0, f"{what}: error {worst:.3f}x the bound"


@pytest.mark.parametrize("dim", [320, 256, 1280, 384])
def test_timestep_embedding_one_row_per_value(dim):
    from cfgpp_b200 import _native as nv
    ts = [0.0, 1.0, 517.37, 83.125, 999.0, 1024.0, 2048.0]
    for t in ts:
        vals = torch.tensor([t], dtype=torch.float32, device=dev)
        out = nv.op_timestep_embedding(vals, 1, dim)
        _check_sincos(f"sincos dim {dim} t {t}", out, vals, dim)
    vals = torch.tensor(ts, dtype=torch.float32, device=dev)
    out = nv.op_timestep_embedding(vals, len(ts), dim)
    _check_sincos(f"sincos dim {dim} {len(ts)} rows", out, vals, dim)


def _check_add_layout(what, tids, seed):
    """The text_time add-embedding input [pooled (PD) | NT time ids x 256]: one launch per id, val_stride NT,
    col_off = PD + j 256; columns outside each slice keep what was there."""
    from cfgpp_b200 import _native as nv
    PD, ATE = 1280, 256
    n, NT = tids.shape
    g = torch.Generator().manual_seed(seed)
    before = rnd(g, n, PD + NT * ATE)
    out = before.clone()
    flat = tids.reshape(-1).contiguous()
    for j in range(NT):
        nv.op_timestep_embedding(flat[j:], n, ATE, out=out, val_stride=NT, col_off=PD + j * ATE)
    torch.cuda.synchronize()
    assert torch.equal(bits(out[:, :PD]), bits(before[:, :PD])), "columns before the time-id slices were written"
    for j in range(NT):
        _check_sincos(f"sincos {what} time id {j}", out[:, PD + j * ATE:PD + (j + 1) * ATE], tids[:, j].contiguous(),
                      ATE)
    narrow = before.clone()[:, :PD + 2 * ATE].contiguous()
    mark = narrow.clone()
    nv.op_timestep_embedding(flat, n, ATE, out=narrow, val_stride=NT, col_off=PD)
    assert torch.equal(bits(narrow[:, PD + ATE:]), bits(mark[:, PD + ATE:])), "columns after the slice were written"


def test_timestep_embedding_sdxl_add_layout():
    """The SDXL base's 6 time ids: original size, crop top-left, target size."""
    tids = torch.tensor([[1024., 1024, 0, 0, 1024, 1024], [768, 1344, 64, 32, 1024, 1024],
                         [517.37, 999, 1, 2048, 896, 1152], [2048, 2048, 0, 0, 2048, 2048]], device=dev)
    _check_add_layout("SDXL", tids, 3)


def test_timestep_embedding_refiner_add_layout():
    """The SDXL refiner's 5 time ids (2560 = 1280 + 5 x 256 input columns): original size, crop top-left and the
    aesthetic score (6 for the positive prompt, 2.5 for the negative, and others)."""
    tids = torch.tensor([[1024., 1024, 0, 0, 6], [1216, 832, 0, 0, 2.5], [1344, 768, 64, 32, 7.25],
                         [517.37, 999, 1, 2048, 0], [2048, 2048, 0, 0, 10]], device=dev)
    assert tids.shape[1] == sdxl_refiner_config().num_time_ids
    _check_add_layout("SDXL refiner", tids, 5)


# ---- small_linear -----------------------------------------------------------------------------------------------

def _linear_ref(x, w, b, addend=None, out_silu=False):
    """(out, out2): t = fp16(x.w + b) in fp64, then fp16(t + addend), out = t or fp16(silu(t)), out2 = fp16(silu(t))."""
    t = (x.double() @ w.double().t() + b.double()).half()
    if addend is not None:
        t = (t.float() + addend.float()).half()
    s = F.silu(t.double()).half()
    return (s if out_silu else t), s


SDXL_TEMB_TOTAL = 2 * 320 + 2 * 640 + 2 * 1280 + 2 * 1280 + 3 * 1280 + 3 * 640 + 3 * 320  # every resnet's time_emb_proj


def temb_total(cfg):
    """Rows of the concatenated time_emb_proj of every resnet (down, mid, up) of a UNet config."""
    ch, lpb = cfg.block_out_channels, cfg.layers_per_block
    return lpb * sum(ch) + 2 * ch[-1] + (lpb + 1) * sum(ch)


REFINER_TEMB_TOTAL = temb_total(sdxl_refiner_config())


@pytest.mark.parametrize("R", [1, 2, 7, 16])
@pytest.mark.parametrize("K,N", [(320, 1000), (1280, 1280), (2816, 1000), (1280, SDXL_TEMB_TOTAL),
                                 # the SDXL refiner: time_embedding.linear_1 / _2, add_embedding.linear_1, time_emb_proj
                                 (384, 1536), (1536, 1536), (2560, 1536), (1536, REFINER_TEMB_TOTAL),
                                 # the CLIP vision towers' visual_projection: ViT-H 1280 -> 1024, ViT-bigG 1664 -> 1280
                                 (1280, 1024), (1664, 1280)])
def test_small_linear(R, K, N):
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(R * 131 + K + N)
    x, w, b = rnd(g, R, K), rnd(g, N, K, scale=K ** -0.5), rnd(g, N, scale=0.5)
    tag = f"small_linear R {R} K {K} N {N}"
    # plain, with out2 = fp16(silu(out))
    out, out2 = nv.op_small_linear(x, w, b, want_out2=True)
    ref, ref2 = _linear_ref(x, w, b)
    gate(tag, out, ref, TOL_GEMM)
    gate(tag + " out2", out2, ref2, TOL_GEMM)
    # out_silu replaces out by what out2 holds without it: same t, same SiLU, bit for bit
    outs, _ = nv.op_small_linear(x, w, b, out_silu=True)
    assert torch.equal(bits(outs), bits(out2)), f"{tag}: out_silu output differs from out2"
    silu_flips = (bits(out2) != bits(F.silu(out.float()).half())).sum().item()
    silu_ulp = ((out2.double() - F.silu(out.double())).abs() / ulp16(F.silu(out.double()))).max().item()
    print(f"[small kernels] {tag}: out2 vs fp16(torch silu(out)): {silu_flips} flips, max {silu_ulp:.3f} ulp")
    assert silu_ulp <= 1.0
    # addend (fp16 add after the rounding) and out_silu
    addend = rnd(g, R, N)
    out, out2 = nv.op_small_linear(x, w, b, addend=addend, out_silu=True, want_out2=True)
    ref, ref2 = _linear_ref(x, w, b, addend, out_silu=True)
    gate(tag + " +addend, out_silu", out, ref, TOL_GEMM)
    # ld_in = 0: one input row broadcast to R rows (time_embedding.linear_2 with the per-row add-embedding)
    x1 = rnd(g, 1, K)
    out, out2 = nv.op_small_linear(x1, w, b, addend=addend, rows=R, want_out2=True)
    ref, ref2 = _linear_ref(x1.expand(R, K), w, b, addend)
    gate(tag + " ld_in 0 +addend", out, ref, TOL_GEMM)
    gate(tag + " ld_in 0 +addend out2", out2, ref2, TOL_GEMM)
    if R == 16:
        full, _ = nv.op_small_linear(x, w, b, addend=addend)
        for r in range(R):
            one, _ = nv.op_small_linear(x[r:r + 1].contiguous(), w, b, addend=addend[r:r + 1].contiguous())
            assert torch.equal(bits(full[r:r + 1]), bits(one)), f"{tag}: row {r} depends on R"


def test_small_linear_rejects_17_rows():
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(17)
    x, w = rnd(g, 17, 320), rnd(g, 64, 320)
    with pytest.raises(nv.NativeError, match="1..16 rows"):
        nv.op_small_linear(x, w, None)


# ---- copy_rows --------------------------------------------------------------------------------------------------

def test_copy_rows():
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(4)
    for src_rows, cols, R, ld, off in ((3, 1280, 8, 2816, 0), (8, 1280, 8, 2816, 0), (1, 256, 5, 1000, 744),
                                       (2, 40, 16, 48, 8)):
        src = rnd(g, src_rows, cols)
        dst = rnd(g, R + 1, ld)
        ref = dst.clone()
        ref[:R, off:off + cols] = src[torch.arange(R, device=dev) % src_rows]
        nv.op_copy_rows(src, dst, R, col_off=off)
        assert torch.equal(bits(dst), bits(ref)), f"copy_rows {src_rows}->{R} rows, {cols} cols at {off}"


# ---- conv_in ----------------------------------------------------------------------------------------------------

def _conv_in_input(z, scale):
    """The conv input as the reference forms it: fp16 z scaled in fp16 arithmetic (fp32 product rounded once), fp32 z
    scaled in fp32 and then cast to fp16 by autocast."""
    if scale is None:
        return z.half()
    if z.dtype == torch.float16:
        return (z.float() * scale).half()
    return (z * torch.tensor(scale, dtype=torch.float32)).half()


@pytest.mark.parametrize("Cout,B,H,W", [(320, 8, 8, 8), (320, 2, 64, 64), (320, 1, 96, 128), (128, 1, 152, 104),
                                        (128, 3, 12, 4), (512, 1, 64, 64), (512, 8, 8, 4), (512, 1, 152, 104),
                                        # the SDXL refiner: 37·384 fp32 of weights and bias, over 48 KB of shared memory
                                        (384, 2, 128, 128), (384, 1, 152, 104), (384, 3, 12, 4)])
def test_conv_in(Cout, B, H, W):
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(Cout + B * H + W)
    w, b = rnd(g, Cout, 4, 3, 3, scale=36 ** -0.5), rnd(g, Cout, scale=0.3)
    wp = w.reshape(Cout, 36).contiguous()
    z32 = (torch.randn(B, 4, H, W, generator=g) * 3).to(dev)
    c_in = 1.0 / math.sqrt(14.6 ** 2 + 1)
    border = border_mask(H, W)
    for zt in (z32.half(), z32):
        for scale in (None, 1.0, c_in):
            sdev = torch.tensor([scale], dtype=torch.float32, device=dev) if scale is not None else None
            out = nv.op_conv_in(zt, wp, b, in_scale=sdev, reps=2)
            assert torch.equal(bits(out[:B]), bits(out[B:])), "conv_in: the two rep copies differ"
            zin = _conv_in_input(zt, scale)
            ref = F.conv2d(zin.double(), w.double(), b.double(), padding=1).half().permute(0, 2, 3, 1)
            tag = f"conv_in Cout {Cout} {B}x{H}x{W} z {str(zt.dtype)[6:]} scale {scale}"
            gate(tag, out[:B], ref, TOL_GEMM)
            gate(tag + " border", out[:B][:, border], ref[:, border], TOL_GEMM)


# ---- conv_out fused with the CFG++ step -------------------------------------------------------------------------

@pytest.mark.parametrize("B,H,W", [(1, 17, 12), (3, 13, 20), (8, 9, 14)])
def test_conv_out_step(B, H, W):
    _conv_out_step_case(B, H, W, 320, B * 100 + H + W)


@pytest.mark.parametrize("B,H,W", [(1, 17, 12), (3, 13, 20), (2, 128, 128)])
def test_conv_out_step_refiner(B, H, W):
    """The SDXL refiner's conv_out (Cin 384: 27 KB of weights in shared memory), the last at its 1024² latent."""
    _conv_out_step_case(B, H, W, 384, B * 100 + H + W + 384)


def _conv_out_step_case(B, H, W, Cin, seed):
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(seed)
    x = (rnd(g, 2 * B, H, W, Cin).float().abs() * 0.7 - 0.2).half()  # roughly GroupNorm + SiLU output
    w, b = rnd(g, 4, Cin, 3, 3, scale=(9 * Cin) ** -0.5), rnd(g, 4, scale=0.2)
    wp = w.permute(0, 2, 3, 1).reshape(4, 9, Cin).contiguous()
    eu, ec, _ = nv.op_conv_out_step(x, wp, b)
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=1).half()
    border = border_mask(H, W)
    for name, got, r in (("eps_uc", eu, ref[:B]), ("eps_c", ec, ref[B:])):
        tag = f"conv_out {B}x{H}x{W} {name}"
        gate(tag, got, r, TOL_GEMM)
        gate(tag + " border", got[:, :, border], r[:, :, border], TOL_GEMM)
    # fused step == the standalone step on the eps the same launch wrote, bit for bit
    lams = torch.linspace(0.3, 7.5, B, dtype=torch.float32, device=dev)
    n_checked = 0
    for k, (method, dt, coef, uses_aux, slots) in enumerate(coef_variants()):
        z0 = (torch.randn(B, 4, H, W, generator=g) * 3).to(dt).to(dev)
        aux0 = torch.randn(B, 4, H, W, generator=g).to(dt).to(dev) if uses_aux else None
        noise = torch.randn(max(slots, 1), B, 4, H, W, generator=g).half().to(dev) if slots else None
        for lam in (None, lams):
            z, aux = z0.clone(), (aux0.clone() if uses_aux else None)
            e_uc, e_c, zt = nv.op_conv_out_step(x, wp, b, method, coef, z, aux=aux, noise=noise, lambdas=lam)
            assert torch.equal(e_uc, eu) and torch.equal(e_c, ec), "the eps of a fused launch differ from STEP_NONE's"
            zs, auxs = z0.clone(), (aux0.clone() if uses_aux else None)
            zts = nv.op_cfgpp_step(e_uc, e_c, method, coef, zs, aux=auxs, noise=noise, lambdas=lam)
            tag = f"conv_out_step {B}x{H}x{W} variant {k} (method {method}, {dt}, bits {coef.second_order}, " \
                  f"{'table' if lam is not None else 'scalar'})"
            assert torch.equal(z, zs) and torch.equal(zt, zts), tag
            if uses_aux:
                assert torch.equal(aux, auxs), tag + " aux"
            n_checked += 1
    print(f"[small kernels] conv_out_step {B}x{H}x{W}: {n_checked} fused step variants bitwise equal to the "
          f"standalone step")


# ---- upsample2x -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,H,W,C", [(2, 5, 7, 8), (1, 9, 13, 320), (3, 16, 24, 320), (2, 8, 3, 1280)])
def test_upsample2x(B, H, W, C):
    from cfgpp_b200 import _native as nv
    x = rnd(torch.Generator().manual_seed(B + H + W + C), B, H, W, C)
    ref = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(bits(nv.op_upsample2x(x)), bits(ref))


# ---- AutoencoderKL helpers --------------------------------------------------------------------------------------

@pytest.mark.parametrize("scaling", [0.18215, 0.13025])
def test_vae_latent_prep(scaling):
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(int(scaling * 1e5))
    w, b = rnd(g, 4, 4, scale=0.5), rnd(g, 4, scale=0.3)
    z32 = (torch.randn(2, 4, 24, 40, generator=g) * 1.2).to(dev)
    for z in (z32.half(), z32):
        out = nv.op_vae_latent_prep(z, scaling, w, b)
        # z / s in z's dtype (fp32 opmath), a true division: a device divisor keeps torch off its reciprocal path
        zs = (z.float() / torch.tensor(scaling, dtype=torch.float32, device=dev)).half()
        ref = (torch.einsum("oc,bchw->bohw", w.double(), zs.double()) + b.double()[None, :, None, None])
        err = ((out.double() - ref).abs() / ulp16(ref)).max().item()
        print(f"[small kernels] vae_latent_prep s {scaling} z {str(z.dtype)[6:]}: max {err:.3f} fp16 ulp")
        assert err <= 1.0


def _softmax_rows(n, g):
    """Score rows (fp16) for the VAE softmax: random, uniform, one dominant score outside the first warp's vectors,
    and scores near +-fp16 max."""
    rows = {}
    rows["random"] = rnd(g, 3, n, scale=30.0)
    rows["uniform"] = torch.full((2, n), 3.0, dtype=torch.float16, device=dev)
    rows["uniform"][1] = -65504.0
    dom = rnd(g, 2, n)
    dom[0, n // 2 + 8 * 40 + 3 if n > 64 else 5] = 60000.0
    dom[1, n - 1] = 300.0
    rows["dominant"] = dom
    big = 65504.0 - 32.0 * torch.randint(0, 6, (2, n), generator=g).float()
    big[1] = -big[1]
    big[1, 7] = 65504.0
    rows["near fp16 max"] = big.half().to(dev)
    return rows


@pytest.mark.parametrize("n", [64, 4096, 16384, 9216, 6144])
def test_vae_row_softmax(n):
    """p = softmax(s / sqrt(512)) per row, against the fp64 softmax of the fp16 scores. The kernel normalises in fp32
    and rounds P once; the gate per element is 1 fp16 ulp of p, or 2^-25 (half the subnormal spacing) below the normal
    range."""
    from cfgpp_b200 import _native as nv
    scale = 1.0 / math.sqrt(512)
    g = torch.Generator().manual_seed(n)
    for kind, s in _softmax_rows(n, g).items():
        ref = torch.softmax(s.double() * scale, dim=1)
        got = nv.op_vae_row_softmax(s.clone(), scale)
        assert torch.isfinite(got).all(), f"softmax n {n} {kind}: inf or NaN"
        err = (got.double() - ref).abs()
        # + 2^-20 p: the fp32 exp2 / sum / normalisation error, which can tip a value sitting on a rounding midpoint
        bound = torch.maximum(ulp16(ref, normal_only=True), torch.full_like(ref, 2.0 ** -25)) + ref * 2.0 ** -20
        worst = (err / bound).max().item()
        sum_err = (got.double().sum(1) - 1).abs().max().item()
        print(f"[small kernels] vae_row_softmax n {n} {kind}: max err/bound {worst:.3f}, max |err| "
              f"{err.max().item():.3e}, row-sum error {sum_err:.3e}")
        assert worst <= 1.0, f"softmax n {n} {kind}: {worst:.3f}x the bound"


@pytest.mark.parametrize("C,B,H,W", [(128, 2, 9, 13), (256, 3, 32, 48), (128, 1, 1024, 1024)])
def test_vae_conv_rgb(C, B, H, W):
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(C + H)
    x = (rnd(g, B, H, W, C).float().abs() * 0.7 - 0.2).half()
    w, b = rnd(g, 3, C, 3, 3, scale=(9 * C) ** -0.5), rnd(g, 3, scale=0.2)
    out = nv.op_vae_conv_rgb(x, w.permute(0, 2, 3, 1).reshape(3, 9, C).contiguous(), b)
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=1).half()
    tag = f"vae_conv_rgb C {C} {B}x{H}x{W}"
    gate(tag, out, ref, TOL_GEMM)
    border = border_mask(H, W)
    gate(tag + " border", out[:, :, border], ref[:, :, border], TOL_GEMM)


@pytest.mark.parametrize("B,H,W", [(2, 40, 24), (1, 1024, 1024)])
def test_vae_image_pad(B, H, W):
    from cfgpp_b200 import _native as nv
    img = (torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(H)) * 2 - 1).to(dev)
    for x in (img.half(), img):
        out = torch.full((B, 4, H, W), float("nan"), dtype=torch.float16, device=dev)
        nv.op_vae_image_pad(x, out=out)
        assert torch.equal(bits(out[:, :3]), bits(x.half())), f"image_pad {str(x.dtype)[6:]}"
        assert bool((bits(out[:, 3]) == 0).all()), "image_pad: the fourth plane is not +0"


def _moments_ref(x, w, b, wq, bq, scaling, noise):
    """The encoder tail as the fp16 module runs under autocast: fp16(conv + b) -> fp16(quant_conv) -> clamp(logvar,
    -30, 20) -> fp16(0.5 logvar) -> fp32 exp -> (mean + std noise) scaling in fp32. Also returns the pre-clamp logvar."""
    m = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=1).half()
    q = (torch.einsum("oc,bchw->bohw", wq.double(), m.double()) + bq.double()[None, :, None, None]).half()
    mean, logvar = q[:, :4], q[:, 4:]
    std = torch.exp((0.5 * logvar.clamp(-30.0, 20.0)).float())
    nz = noise.float() if noise is not None else torch.zeros_like(std)
    return (mean.float() + std * nz) * torch.tensor(scaling, dtype=torch.float32), logvar


# observed 0 (bit-identical at these seeds); one logvar rounding flip near 25 moves std by 0.8%, ≈2.5e-4 of rel-L2
TOL_MOMENTS = 5e-4


@pytest.mark.parametrize("C,B,H,W", [(128, 2, 12, 20), (512, 1, 33, 17), (512, 2, 16, 16)])
def test_vae_moments_sample(C, B, H, W):
    """quant_conv biases put the four logvar channels around -35, -28, 19 and 25, so some pixels sit below -30 and
    above 20; clamped pixels are checked on their own."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(C + B + H)
    scaling = 0.13025
    x = (rnd(g, B, H, W, C).float().abs() * 0.7 - 0.2).half()
    w, b = rnd(g, 8, C, 3, 3, scale=(9 * C) ** -0.5), rnd(g, 8, scale=0.2)
    wq = rnd(g, 8, 8, scale=0.4)
    wq[4:] = (wq[4:].float() * 5).half()
    bq = torch.tensor([0.1, -0.2, 0.05, 0.3, -35.0, -28.0, 19.0, 25.0], dtype=torch.float16, device=dev)
    wp = w.permute(0, 2, 3, 1).reshape(8, 9, C).contiguous()
    noise = rnd(g, B, 4, H, W)
    for nz in (None, noise):
        out = nv.op_vae_moments_sample(x, wp, b, wq, bq, scaling, noise=nz)
        ref, logvar = _moments_ref(x, w, b, wq, bq, scaling, nz)
        tag = f"vae_moments C {C} {B}x{H}x{W} {'noise' if nz is not None else 'mean'}"
        gate(tag, out, ref, TOL_MOMENTS)
        low, high = logvar < -30.0, logvar > 20.0
        assert low.any() and high.any() and (~(low | high)).any(), "the biases no longer reach both clamp bounds"
        gate(tag + f" logvar < -30 ({low.sum().item()} px)", out[low], ref[low], TOL_MOMENTS)
        gate(tag + f" logvar > 20 ({high.sum().item()} px)", out[high], ref[high], TOL_MOMENTS)


# ---- CLIP text tower kernels ------------------------------------------------------------------------------------

def test_clip_embed_and_gather_rows():
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(77)
    vocab, T, D, B = 49408, 77, 768, 3
    tok, pos = rnd(g, vocab, D), rnd(g, T, D, scale=0.1)
    ids = torch.randint(0, vocab, (B * T,), generator=g, dtype=torch.int32)
    ids[0], ids[1], ids[T + 5], ids[-1] = 0, vocab - 1, vocab - 1, 0
    ids = ids.to(dev)
    out = nv.op_clip_embed(ids, tok, pos)
    ref = (tok[ids.long()].float() + pos[torch.arange(B * T, device=dev) % T].float()).half()
    assert torch.equal(bits(out), bits(ref)), "clip_embed"
    x = rnd(g, B * T, D)
    index = torch.tensor([0, T - 1, 41], dtype=torch.int32, device=dev)
    got = nv.op_clip_gather_rows(x, index, T)
    assert torch.equal(bits(got), bits(x[torch.arange(B, device=dev) * T + index.long()])), "clip_gather_rows"


@pytest.mark.parametrize("B,T,heads", [(1, 1, 12), (2, 2, 12), (16, 77, 12), (4, 77, 20), (2, 128, 20),
                                       (1, 77, 16), (8, 77, 16), (3, 128, 16)])  # 16 heads: ViT-H
def test_clip_attention(B, T, heads):
    from cfgpp_b200 import _native as nv
    D = 64 * heads
    g = torch.Generator().manual_seed(B * T + heads)
    qkv = rnd(g, B * T, 3 * D, scale=1.5)
    out = nv.op_clip_attention(qkv, B, T, heads)
    q, k, v = qkv.double().view(B, T, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / 8.0
    s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device=dev).triu(1), float("-inf"))
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * T, D)
    tag = f"clip_attention B {B} T {T} heads {heads}"
    gate(tag, out, ref.half(), TOL_GEMM)
    row0 = qkv.view(B, T, 3 * D)[:, 0, 2 * D:]
    assert torch.equal(bits(out.view(B, T, D)[:, 0]), bits(row0)), f"{tag}: row 0 is not v[0]"


def test_clip_attention_rejects_129_tokens():
    from cfgpp_b200 import _native as nv
    qkv = torch.zeros(129, 3 * 768, dtype=torch.float16, device=dev)
    with pytest.raises(nv.NativeError, match="at most 128 tokens"):
        nv.op_clip_attention(qkv, 1, 129, 12)


def _all_finite_fp16():
    b = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    x = b.view(torch.float16)
    return x[torch.isfinite(x)].contiguous().to(dev)


@pytest.mark.parametrize("mode", [0, 1])
def test_clip_activation_every_fp16_input(mode):
    """All 63,488 finite fp16 inputs, against torch on the same GPU: mode 0 against transformers' QuickGELUActivation
    on an fp16 module (`x * torch.sigmoid(1.702 * x)`, three fp16 ops), mode 1 against F.gelu on fp16 (fp32 erf
    formula, one rounding). Both bit for bit."""
    from cfgpp_b200 import _native as nv
    x = _all_finite_fp16()
    assert x.numel() == 63488
    ref = x * torch.sigmoid(1.702 * x) if mode == 0 else F.gelu(x)
    got = nv.op_clip_activation(x.clone(), mode)
    diff = bits(got) != bits(ref)
    nd = int(diff.sum().item())
    if nd:
        u = ((got[diff].double() - ref[diff].double()).abs() / ulp16(ref[diff].double())).max().item()
        print(f"[small kernels] clip_act mode {mode}: {nd} of {x.numel()} inputs differ, max {u:.1f} ulp; "
              f"first at x = {x[diff][:4].tolist()}")
    else:
        print(f"[small kernels] clip_act mode {mode}: all {x.numel()} finite fp16 inputs bit-exact")
    assert nd == 0
