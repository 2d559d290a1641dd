"""Kernel-level parity (through the C ABI) against torch fp32 references of the same op, with the reference's
rounding points (fp16(acc+bias) then fp16 add of the residual / time embedding).
Gates are ~5x the error observed on the GPU (printed by every test; `pytest -s` shows them): GEMM / conv observe ~3e-5
(both sides round the same fp32 sum to fp16, so only accumulation-order flips of the last bit remain) -> 2e-4.
Attention and the norms are pinned element by element against fp64 in `test_gpu_attention.py` and
`test_gpu_norms.py`."""
import pytest
import torch

from helpers import rel_l2

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _fp32_refs():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


TOL_GEMM = 2e-4


def gate(what, got, ref, tol):
    e = rel_l2(got, ref)
    print(f"[kernel parity] {what}: rel-L2 {e:.3e} (gate {tol:.1e})")
    assert e < tol, f"{what}: rel-L2 {e:.3e} >= {tol:.1e}"


def rnd(g, *s, scale=1.0, shift=0.0):
    return (torch.randn(*s, generator=g) * scale + shift).half().to(dev)


def ref_linear(a, w, bias, addend, rpg):
    acc = a.float() @ w.float().t()
    if bias is not None:
        acc = acc + bias.float()
    t = acc.half()
    if addend is not None:
        ad = addend.float()
        if rpg > 1:
            ad = ad.repeat_interleave(rpg, dim=0)[: a.shape[0]]
        t = (t.float() + ad).half()
    return t


@pytest.mark.parametrize("M,N,K,hb,ha,bn", [
    (128, 64, 64, False, 0, 64), (256, 256, 256, True, 0, 256), (256, 320, 320, True, 1, 160),
    (308, 1280, 2048, False, 0, 0), (4096, 1280, 1280, True, 1, 0), (2048, 320, 960, True, 1024, 0),
    (1000, 200, 192, True, 1, 128), (16384, 1920, 640, False, 0, 0), (1, 64, 64, True, 0, 0), (77, 8, 64, False, 0, 0)])
def test_linear(M, N, K, hb, ha, bn):
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(M * 7 + N)
    a, w = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5)
    bias = rnd(g, N) if hb else None
    addend = rnd(g, M, N) if ha == 1 else (rnd(g, (M + ha - 1) // ha, N) if ha > 1 else None)
    out = nv.op_linear(a, w, bias, addend, ha if ha > 1 else 1, force_bn=bn)
    gate(f'linear {M}x{N}x{K}', out, ref_linear(a, w, bias, addend, ha), TOL_GEMM)


@pytest.mark.parametrize("force_streamk", [False, True])
@pytest.mark.parametrize("M,N,K,geglu_like", [(4096, 1280, 1280, False), (4096, 1280, 5120, False),
                                              (4096, 3840, 1280, False), (2048, 640, 2560, False),
                                              (8192, 1280, 1280, False), (5000, 1280, 640, False)])
def test_linear_streamk_shapes_and_repeatability(M, N, K, geglu_like, force_streamk):
    """Shapes whose tile count is not a multiple of the CTA count CAN take the stream-K remainder path (partials
    parked in the workspace by other CTAs, self-resetting flags; on by default for the convolutions, off for linear
    layers unless `force_streamk` is set, so the forced cases cover the split's partial / fix-up path): result vs the
    fp32 reference, and 12 back-to-back launches must be bit-identical (fixed summation order; flags re-armed by the
    kernel itself)."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(M + N + K)
    a, w, bias, res = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5), rnd(g, N), rnd(g, M, N)
    first = nv.op_linear(a, w, bias, res, 1, force_streamk=force_streamk)
    gate(f'linear(force_streamk={force_streamk}) {M}x{N}x{K}', first, ref_linear(a, w, bias, res, 1), TOL_GEMM)
    for _ in range(12):
        assert torch.equal(nv.op_linear(a, w, bias, res, 1, force_streamk=force_streamk), first)


def test_linear_dual_source_and_geglu():
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(5)
    a1, a2 = rnd(g, 1024, 640), rnd(g, 1024, 320)
    w, bias = rnd(g, 320, 960, scale=960 ** -0.5), rnd(g, 320)
    out = nv.op_linear(a1, w, bias, None, 1, a2=a2)
    gate('linear dual-source', out, ref_linear(torch.cat([a1, a2], 1), w, bias, None, 1), TOL_GEMM)
    M, Cc = 512, 640
    inner = 4 * Cc
    a, w, b = rnd(g, M, Cc), rnd(g, 2 * inner, Cc, scale=Cc ** -0.5), rnd(g, 2 * inner)
    idx = []
    for t in range(inner // 128):
        idx += list(range(t * 128, t * 128 + 128)) + list(range(inner + t * 128, inner + t * 128 + 128))
    idx = torch.tensor(idx, device=dev)
    out = nv.op_linear(a, w[idx].contiguous(), b[idx].contiguous(), geglu=True)
    h = (a.float() @ w.float().t() + b.float()).half()
    ref = (h[:, :inner].float() * torch.nn.functional.gelu(h[:, inner:].float()).half().float()).half()
    gate('geglu', out, ref, TOL_GEMM)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(4, 128, 128, 320, 320), (4, 64, 64, 640, 640), (2, 32, 32, 128, 128),
                                            (1, 16, 16, 64, 64), (2, 96, 128, 64, 64)])
def test_conv3x3_stride2(B, H, W, Cin, Cout):
    """Downsample2D (3x3, stride 2, pad 1): the A tiles come through a tensor map with element strides 2 — the first
    row / column of taps starts at input coordinate -1 (TMA zero fill), every second pixel is fetched."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(H + Cin)
    x, w, bias = rnd(g, B, Cin, H, W), rnd(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5), rnd(g, Cout)
    out = nv.op_conv3x3_s2(x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous(),
                           bias).reshape(-1, Cout)
    ref = torch.nn.functional.conv2d(x.float(), w.float(), bias.float(), stride=2, padding=1).half()
    gate(f'conv3x3 stride 2 {B}x{H}x{W} {Cin}->{Cout}', out, ref.permute(0, 2, 3, 1).reshape(-1, Cout), TOL_GEMM)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 256, 256, 128, 128), (2, 128, 128, 256, 256), (2, 32, 32, 64, 64),
                                            (1, 64, 128, 128, 128)])
def test_conv3x3_stride2_pad_after(B, H, W, Cin, Cout):
    """The AutoencoderKL encoder's Downsample2D: F.pad(x, (0, 1, 0, 1)) then an un-padded stride-2 conv — the same
    stride-2 tensor map started AT the pixel, the zero row / column after the image being the TMA's out-of-bounds fill."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(H + Cin + 1)
    x, w, bias = rnd(g, B, Cin, H, W), rnd(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5), rnd(g, Cout)
    out = nv.op_conv3x3_s2(x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous(),
                           bias, pad=0).reshape(-1, Cout)
    ref = torch.nn.functional.conv2d(torch.nn.functional.pad(x.float(), (0, 1, 0, 1)), w.float(), bias.float(), stride=2).half()
    assert ref.shape[-2:] == (H // 2, W // 2)
    gate(f'conv3x3 stride 2 pad-after {B}x{H}x{W} {Cin}->{Cout}', out, ref.permute(0, 2, 3, 1).reshape(-1, Cout), TOL_GEMM)


def test_conv3x3_streamk_repeatable():
    """The conv shapes of the 1280-channel level take the stream-K split by default: 10 launches, bit-identical."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(11)
    x, w, bias = rnd(g, 4, 32, 32, 1280), rnd(g, 1280, 9 * 1280, scale=(9 * 1280) ** -0.5), rnd(g, 1280)
    res = rnd(g, 4 * 32 * 32, 1280)
    first = nv.op_conv3x3(x, w, bias, res, 1)
    for _ in range(10):
        assert torch.equal(nv.op_conv3x3(x, w, bias, res, 1), first)


@pytest.mark.parametrize("B,H,W,Cin,Cout,ht,hr", [
    (1, 32, 32, 64, 64, False, False), (2, 64, 64, 128, 128, True, False), (4, 16, 16, 128, 256, False, True),
    (2, 8, 8, 128, 128, True, False), (1, 128, 128, 320, 320, True, False), (4, 32, 32, 1280, 1280, False, True),
    # non-square / non-power-of-two H (landscape aspect buckets), W > 128 row segments (VAE decoder levels)
    (2, 96, 128, 64, 128, True, False), (1, 24, 32, 128, 128, False, True), (3, 6, 64, 64, 64, False, False),
    (1, 40, 256, 64, 64, False, True), (1, 16, 1024, 64, 64, True, False),
    # fewer tiles than clusters with a long K: every tile is split over ~5 clusters (stream-K with 4-5 partials)
    (8, 8, 8, 1280, 1280, True, False), (8, 8, 8, 2560, 1280, False, True)])
def test_conv3x3(B, H, W, Cin, Cout, ht, hr):
    """Zero padding comes from TMA out-of-bounds fill; edge pixels are therefore the interesting ones."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(H * 3 + Cin)
    x, w, bias = rnd(g, B, Cin, H, W), rnd(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5), rnd(g, Cout)
    addend, rpg = None, 1
    if ht:
        addend, rpg = rnd(g, B, Cout), H * W
    elif hr:
        addend = rnd(g, B * H * W, Cout)
    out = nv.op_conv3x3(x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous(),
                        bias, addend, rpg).reshape(B * H * W, Cout)
    ref = torch.nn.functional.conv2d(x.float(), w.float(), bias.float(), padding=1).half()
    ref = ref.permute(0, 2, 3, 1).reshape(B * H * W, Cout)
    if ht:
        ref = (ref.float() + addend.float().repeat_interleave(H * W, 0)).half()
    elif hr:
        ref = (ref.float() + addend.float()).half()
    gate(f'conv3x3 {B}x{H}x{W} {Cin}->{Cout}', out, ref, TOL_GEMM)
    edge = torch.zeros(B, H, W, dtype=torch.bool, device=dev)
    edge[:, 0], edge[:, -1], edge[:, :, 0], edge[:, :, -1] = True, True, True, True
    gate('conv3x3 edge pixels', out[edge.reshape(-1)], ref[edge.reshape(-1)], TOL_GEMM)
