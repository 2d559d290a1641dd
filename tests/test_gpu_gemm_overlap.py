"""The GEMM epilogue hand-off under pressure: the MMA warps write a tile's fp16 result into the staging tile and go on to
the next tile's main loop, while the service warps store it, refill the staging tile with the next residual and stage
the next tiles' vectors. At K = 64 and 128 (one and two k-blocks) the main loop is far shorter than that work, so every
tile waits on "staging free" and on its vectors, and every CTA walks at least 8 tiles, so both vector buffers and both
staged barriers turn over several times.

Integer operands (test_gpu_gemm.py's Family A): each launch is bit-identical to the fp16 rounding chain of the exact
result, in every epilogue variant, and 10 back-to-back launches are bit-identical to each other."""
import pytest
import torch

from test_gpu_gemm import check_exact, dev, gen, geglu_int_operands, int_act, int_vec, int_weight, linear_kblocks, run_linear

pytestmark = pytest.mark.gpu

REPEATS = 10


def tiles_rows(bn, n, per_cta=8):
    """M (a multiple of 128) that gives every CTA at least `per_cta` tiles of width bn over n columns."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    n_blocks = (n + bn - 1) // bn
    m_blocks = (per_cta * sms + n_blocks - 1) // n_blocks
    return 128 * m_blocks


def repeat_identical(run, first, what):
    for i in range(REPEATS):
        again = run()
        assert all(torch.equal(x, y) for x, y in zip(again, first)), f"{what}: launch {i + 1} differs from the first"


def schedule_per_cta(a, w, **kw):
    from cfgpp_b200 import _native as nv
    s = nv.linear_schedule(a, w, **kw)
    return s, s["tiles"] / s["grid"]


@pytest.mark.parametrize("K", [64, 128])
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("mode", ["none", "bias", "residual", "in_place", "temb_staged", "temb_rows"])
def test_overlap_plain(K, bn, mode):
    from cfgpp_b200 import _native as nv
    N = 1280
    M = tiles_rows(bn, N)
    g = gen(1000 * K + bn + len(mode))
    a, w = int_act(g, M, K), int_weight(g, N, K)
    bias = int_vec(g, N) if mode != "none" else None
    addend, rpg = None, 1
    if mode in ("residual", "in_place"):
        addend = int_vec(g, M, N)
    elif mode.startswith("temb"):
        rpg = 256 if mode == "temb_staged" else 48
        addend = int_vec(g, (M + rpg - 1) // rpg, N)
    s, per_cta = schedule_per_cta(a, w, bias=bias, addend=addend, add_rows_per_group=rpg, force_bn=bn)
    assert s["bn"] == bn and per_cta >= 8 and not s["streamk"], s
    what = f"overlap {M}x{N}x{K} BN{bn} {mode}"
    in_place = mode == "in_place"
    add0 = addend.clone() if in_place else addend
    first, _ = run_linear(what, a, w, bias=bias, addend=addend, rpg=rpg, force_bn=bn, in_place=in_place)
    first = first.clone()

    def run():
        if in_place:
            addend.copy_(add0)
        return (nv.op_linear(a, w, bias, addend, rpg, force_bn=bn, out=addend if in_place else None),)

    repeat_identical(run, (first,), what)


@pytest.mark.parametrize("K", [64, 128])
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("mode", ["none", "residual", "temb_staged"])
def test_overlap_rowstats(K, bn, mode):
    """Row statistics of integer outputs: every partial sum is an integer below 2^24, so the fp32 sums are exact."""
    from cfgpp_b200 import _native as nv
    N = 1280
    M = tiles_rows(bn, N)
    g = gen(2000 * K + bn + len(mode))
    a, w, bias = int_act(g, M, K), int_weight(g, N, K, nnz=32), int_vec(g, N)
    addend, rpg = None, 1
    if mode == "residual":
        addend = int_vec(g, M, N)
    elif mode == "temb_staged":
        rpg = 256
        addend = int_vec(g, M // rpg + 1, N)
    run = lambda: nv.op_linear_stats(a, w, bn, bias, addend, rpg)
    first = run()
    out, stats = first
    what = f"overlap rowstats {M}x{N}x{K} BN{bn} {mode}"
    check_exact(what, out, linear_kblocks(a), w, M, bias, addend, rpg)
    half = bn // 2
    o = out.double()
    exact = torch.stack([torch.stack([o[:, p * half:(p + 1) * half].sum(1), (o[:, p * half:(p + 1) * half] ** 2).sum(1)], 1)
                         for p in range(stats.shape[0])])
    assert exact.abs().max().item() < 2 ** 24
    assert torch.equal(stats, exact.float()), f"{what}: statistics differ from the exact sums"
    repeat_identical(run, first, what)


@pytest.mark.parametrize("K", [64, 128])
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("parts", [2, 8])
def test_overlap_lnfold(K, bn, parts):
    """LayerNorm-fold consumer with statistics of mean 0 and variance 1 (eps 0): rstd = 1 and rstd·mean = 0, so
    out = fp16(acc + t_n) of integers, exact. The `parts` partials are summed by the service warps."""
    from cfgpp_b200 import _native as nv
    N = 1280
    M = tiles_rows(bn, N)
    g = gen(3000 * K + bn + parts)
    h, wf = int_act(g, M, K), int_weight(g, N, K)
    s = int_vec(g, N).float()
    t = int_vec(g, N).float()
    stats = torch.zeros(parts, M, 2, device=dev)
    stats[:, :, 1] = K / parts  # Σx = 0, Σx² = C: mean 0, variance 1
    run = lambda: (nv.op_linear_lnfold(h, wf, s, t, stats, eps=0.0, force_bn=bn),)
    first = run()
    what = f"overlap lnfold {M}x{N}x{K} BN{bn} parts {parts}"
    check_exact(what, first[0], linear_kblocks(h), wf, M, t.half())
    repeat_identical(run, first, what)


@pytest.mark.parametrize("K", [64, 128])
def test_overlap_geglu(K):
    from cfgpp_b200 import _native as nv
    N = 8 * K
    M = tiles_rows(256, N)
    g = gen(4000 + K)
    a, wp, bp = geglu_int_operands(g, M, K)
    first, s = run_linear(f"overlap geglu {M}x{4 * K}x{K}", a, wp, bias=bp, geglu=True)
    assert s["tiles"] / s["grid"] >= 8, s
    first = first.clone()
    repeat_identical(lambda: (nv.op_linear(a, wp, bp, geglu=True),), (first,), f"overlap geglu {M}x{4 * K}x{K}")


@pytest.mark.parametrize("mode", ["bias", "residual"])
def test_overlap_streamk_forced(mode):
    """The forced stream-K split (pieces of >= 2 k-blocks need K = 512 here): the finishing pieces go through the same
    hand-off, the parking pieces take none."""
    from cfgpp_b200 import _native as nv
    N, K, bn = 1024, 512, 128
    M = 128 * 140  # 1120 tiles: 64 left over after 8 rounds of 132 CTAs
    g = gen(5000 + len(mode))
    a, w, bias = int_act(g, M, K), int_weight(g, N, K), int_vec(g, N)
    addend = int_vec(g, M, N) if mode == "residual" else None
    first, s = run_linear(f"overlap stream-K {M}x{N}x{K}", a, w, bias=bias, addend=addend, force_bn=bn,
                          force_streamk=True, expect_sk=True)
    first = first.clone()
    repeat_identical(lambda: (nv.op_linear(a, w, bias, addend, force_bn=bn, force_streamk=True),), (first,),
                     f"overlap stream-K {M}x{N}x{K} {mode}")
