"""The implicit-GEMM 3x3 convolution's two A-tile modes, at kernel level through `op_conv3x3_ex`.

The tiled mode fetches the 128 output pixels of a tile as one 4-D TMA box; the im2col mode walks them through an im2col
tensor map that wraps across row and image ends, so it addresses any H, W. Both fill the same swizzled smem tile in the
same k order, so on every shape the tiled mode can address, forcing im2col must give a bit-identical result. Every
result is also gated element by element against the fp64 reference in the kernel's k order, within the accumulation
bound of `test_gpu_gemm.py` (edge pixels, which read the zero fill, included)."""
import pytest
import torch

from test_gpu_gemm import check_bound, conv_kblocks

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


def rnd(g, *s, scale=1.0):
    return (torch.randn(*s, generator=g) * scale).half().to(dev)


def make_case(seed, B, H, W, Cin, Cout, stride, addend_kind):
    """NCHW input / weight, their NHWC / packed forms, bias and the addend ('temb': one row per image, 'res': a full
    residual, None)."""
    g = torch.Generator().manual_seed(seed)
    x, w, bias = rnd(g, B, Cin, H, W), rnd(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5), rnd(g, Cout)
    Ho, Wo = H // stride, W // stride
    addend, rpg = None, 1
    if addend_kind == "temb":
        addend, rpg = rnd(g, B, Cout), Ho * Wo
    elif addend_kind == "res":
        addend = rnd(g, B * Ho * Wo, Cout)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    w_packed = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    return x, w, bias, addend, rpg, x_nhwc, w_packed


def gate(what, out, case, stride, pad):
    """Every element of out within the per-element bound of the fp64 reference (the launch's own schedule decides
    whether the stream-K term applies)."""
    from cfgpp_b200 import _native as nv
    _, _, bias, addend, rpg, x_nhwc, w_packed = case
    sched = nv.conv3x3_schedule(x_nhwc, w_packed, bias, addend, rpg, stride=stride, pad=pad)
    check_bound(f"[conv geometry] {what}", out, conv_kblocks(x_nhwc, stride, pad), w_packed, out.shape[0], bias,
                addend, rpg, sched)


def run(nv, case, stride, pad, force_im2col):
    x, w, bias, addend, rpg, x_nhwc, w_packed = case
    out = nv.op_conv3x3_ex(x_nhwc, w_packed, bias, addend, rpg, stride=stride, pad=pad, force_im2col=force_im2col)
    return out.reshape(-1, w_packed.shape[0])


# ---- bitwise mode equivalence on tiled-addressable shapes ---------------------------------------------------------
# every shape of test_gpu_gemm.test_conv3x3 (the last three take the stream-K split), stride 1 / pad 1
TILED_S1 = [(1, 32, 32, 64, 64), (2, 64, 64, 128, 128), (4, 16, 16, 128, 256), (2, 8, 8, 128, 128),
            (1, 128, 128, 320, 320), (4, 32, 32, 1280, 1280), (2, 96, 128, 64, 128), (1, 24, 32, 128, 128),
            (3, 6, 64, 64, 64), (1, 40, 256, 64, 64), (1, 16, 1024, 64, 64), (8, 8, 8, 1280, 1280),
            (8, 8, 8, 2560, 1280)]
# the stride-2 cases of test_gpu_gemm (pad 1: Downsample2D; pad 0: the AutoencoderKL encoder's pad-after)
TILED_S2 = [(4, 128, 128, 320, 320, 1), (4, 64, 64, 640, 640, 1), (2, 32, 32, 128, 128, 1), (1, 16, 16, 64, 64, 1),
            (2, 96, 128, 64, 64, 1), (1, 256, 256, 128, 128, 0), (2, 128, 128, 256, 256, 0), (2, 32, 32, 64, 64, 0),
            (1, 64, 128, 128, 128, 0)]


@pytest.mark.parametrize("addend_kind", [None, "temb", "res"])
@pytest.mark.parametrize("B,H,W,Cin,Cout", TILED_S1)
def test_im2col_equals_tiled_stride1(B, H, W, Cin, Cout, addend_kind):
    from cfgpp_b200 import _native as nv
    case = make_case(H * 3 + Cin + W, B, H, W, Cin, Cout, 1, addend_kind)
    tiled = run(nv, case, 1, 1, False)
    im2col = run(nv, case, 1, 1, True)
    assert torch.equal(tiled, im2col), f"{B}x{H}x{W} {Cin}->{Cout} addend={addend_kind}: modes differ"
    gate(f"tiled {B}x{H}x{W} {Cin}->{Cout} addend={addend_kind}", tiled, case, 1, 1)


@pytest.mark.parametrize("addend_kind", [None, "temb", "res"])
@pytest.mark.parametrize("B,H,W,Cin,Cout,pad", TILED_S2)
def test_im2col_equals_tiled_stride2(B, H, W, Cin, Cout, pad, addend_kind):
    from cfgpp_b200 import _native as nv
    case = make_case(H + Cin + pad, B, H, W, Cin, Cout, 2, addend_kind)
    tiled = run(nv, case, 2, pad, False)
    im2col = run(nv, case, 2, pad, True)
    assert torch.equal(tiled, im2col), f"s2 pad {pad} {B}x{H}x{W} {Cin}->{Cout} addend={addend_kind}: modes differ"
    gate(f"tiled s2 pad {pad} {B}x{H}x{W} {Cin}->{Cout} addend={addend_kind}", tiled, case, 2, pad)


# ---- geometries only the im2col A tile addresses, against the fp64 reference ------------------------------------------
def check_new_geometry(B, H, W, Cin, Cout, stride, pad, addend_kind):
    from cfgpp_b200 import _native as nv
    case = make_case(B * 1000 + H * 7 + W + Cin + stride + pad, B, H, W, Cin, Cout, stride, addend_kind)
    assert nv.conv3x3_schedule(case[5], case[6], stride=stride, pad=pad)["a_mode"] == "im2col"
    out = run(nv, case, stride, pad, False)
    gate(f"s{stride} pad {pad} {B}x{H}x{W} {Cin}->{Cout} addend={addend_kind}", out, case, stride, pad)
    return out


# odd and even widths, none of them tiled-addressable at these heights
WIDTHS = [1, 3, 7, 12, 20, 24, 26, 38, 52, 76, 80, 96, 104, 144, 152, 168, 192, 208, 304, 608, 1216]


@pytest.mark.parametrize("W", WIDTHS)
def test_new_widths(W):
    H = 5 if W <= 208 else 3  # H * W: below 128 for the narrow ones, above and not a multiple of 128 for the wide ones
    check_new_geometry(2, H, W, 64, 64, 1, 1, "temb")


@pytest.mark.parametrize("B,H,W,Cin,Cout,addend_kind", [
    (1, 5, 7, 64, 64, None),            # H·W = 35 < 128: one tile holds the whole batch and runs past it
    (3, 11, 13, 128, 64, "temb"),       # H·W = 143 > 128, not a multiple: tiles straddle images mid-row
    (16, 9, 12, 64, 128, "temb"),       # B = 16, H·W = 108: nearly every tile holds two images' rows
    (16, 13, 13, 64, 64, "res"),        # B·H·W = 2704 = 21·128 + 16: the last tile walks past the last image
    (5, 104, 152, 64, 64, "temb"),      # an SDXL bucket latent, five images
    (2, 152, 104, 320, 320, "res"),
    (1, 96, 168, 128, 128, None),
    (2, 80, 192, 64, 128, "temb"),
    (2, 64, 96, 320, 320, "temb"),      # SD v1.5 512 x 768
    (2, 12, 8, 64, 64, "temb"),         # its lowest level (96 x 64 -> 12 x 8)
])
def test_new_geometries(B, H, W, Cin, Cout, addend_kind):
    check_new_geometry(B, H, W, Cin, Cout, 1, 1, addend_kind)


@pytest.mark.parametrize("B,H,W,Cin,Cout,addend_kind", [
    (2, 13, 19, 1280, 1280, "temb"),    # the 1280-channel level of a bucket: stream-K with partials
    (1, 26, 38, 2560, 1280, "res"),     # Cin 2560 (an up-block's concat input)
    (4, 12, 10, 2560, 640, "temb"),
])
def test_new_geometries_streamk(B, H, W, Cin, Cout, addend_kind):
    check_new_geometry(B, H, W, Cin, Cout, 1, 1, addend_kind)


@pytest.mark.parametrize("pad", [1, 0])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 104, 152, 64, 64), (1, 152, 104, 128, 128), (3, 24, 20, 64, 64),
                                            (2, 52, 76, 320, 320), (1, 208, 304, 128, 128), (2, 6, 10, 64, 64)])
def test_new_geometries_stride2(B, H, W, Cin, Cout, pad):
    check_new_geometry(B, H, W, Cin, Cout, 2, pad, None)


def test_temb_on_tiles_straddling_images_mid_row():
    """Each image gets its own time-embedding row, also in tiles that hold the end of one image and the start of the
    next part-way through a row: per image, the result equals that image run alone."""
    from cfgpp_b200 import _native as nv
    B, H, W, C = 6, 7, 26, 64  # H·W = 182: the tile boundaries fall mid-row
    x, w, bias, addend, rpg, x_nhwc, w_packed = make_case(77, B, H, W, C, C, 1, "temb")
    out = nv.op_conv3x3_ex(x_nhwc, w_packed, bias, addend, rpg)
    for b in range(B):
        one = nv.op_conv3x3_ex(x_nhwc[b:b + 1].contiguous(), w_packed, bias, addend[b:b + 1].contiguous(), rpg)
        assert torch.equal(out[b], one[0]), f"image {b}"


def test_im2col_streamk_repeatable():
    """Ten launches at a stream-K im2col shape are bit-identical (fixed summation order of the parked partials)."""
    from cfgpp_b200 import _native as nv
    x, w, bias, addend, rpg, x_nhwc, w_packed = make_case(11, 2, 13, 19, 1280, 1280, 1, "res")
    first = nv.op_conv3x3_ex(x_nhwc, w_packed, bias, addend, rpg)
    for _ in range(10):
        assert torch.equal(nv.op_conv3x3_ex(x_nhwc, w_packed, bias, addend, rpg), first)
