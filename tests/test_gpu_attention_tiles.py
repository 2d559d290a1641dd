"""The 128-row tile geometry of the head-dim-64 attention kernel `attn64_kernel` / `attn64_ip_kernel` (`attention.cu`):
one CTA per 128 query rows (two consumer warpgroups of 64), K / V in 128-row tiles through a 4-stage ring.

The per-element gate is `test_gpu_attention.check` (|out − ref| ≤ E against fp64). The cases sit at the boundaries
of that geometry: query counts around 128 and 256 (a warpgroup with no valid rows, a last tile of 1 row), KV counts
around 128-row tiles, enough tiles to wrap the ring and flip its parity, and head dims 64 and 40 (padded to 64)."""
import math

import pytest
import torch

from test_gpu_attention import check, family, fused, gen, heads, padded

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

NQ = (127, 128, 129, 255, 257, 385)
NKV = (255, 256, 257, 383, 385, 1025)
FAMILIES = ("flat", "peaked", "rising", "hot_last", "extreme")


@pytest.mark.parametrize("hd", (64, 40))
@pytest.mark.parametrize("name", FAMILIES)
def test_tile_boundaries(name, hd):
    """Every family at every (Nq, Nkv) of the sweep, B = 1 and 3, two heads; q / k / v slices of one fused buffer
    when Nq = Nkv, k / v slices of one KV buffer otherwise."""
    H, hdp = 2, padded(hd)
    g = gen(FAMILIES.index(name) * 1000 + hd + 71)
    for B in (1, 3):
        for Nq in NQ:
            for Nkv in NKV:
                q, k, v = (heads(t, hdp) for t in family(name, g, B, Nq, Nkv, H, hd))
                if Nq == Nkv:
                    q, k, v = fused(q, k, v)
                else:
                    k, v = fused(k, v)
                check(f"{name} hd{hd} B{B} {Nq}x{Nkv}", q, k, v, H, hd)


@pytest.mark.parametrize("hd", (64, 40))
def test_known_answer_one_hot_128(hd):
    """One key ≈ 70 nats above the rest: the output is its value row bit for bit. The hot key sits at column 0, at
    127 and 128 (the two sides of the first 128-column tile) and at the last valid column of a partial last tile."""
    from cfgpp_b200 import _native as nv
    B, H, Nq, hdp = 2, 2, 257, padded(hd)
    g = gen(hd + 97)
    u = torch.ones(H, hd, device=dev)
    for Nkv in (200, 300, 385):
        for hot in sorted({0, 127, 128, Nkv - 1}):
            q = u + 0.05 * torch.randn(B, Nq, H, hd, generator=g, device=dev)
            k = 0.5 * torch.randn(B, Nkv, H, hd, generator=g, device=dev)
            k[:, hot] = u * (70 / math.sqrt(hd))
            v = heads(torch.randn(B, Nkv, H, hd, generator=g, device=dev), hdp)
            k, v = fused(heads(k, hdp), v)
            out = nv.op_attention(heads(q, hdp), k, v, H, head_dim=hd)
            want = v[:, hot:hot + 1].expand(B, Nq, H * hdp)
            assert torch.equal(out, want), f"hd{hd} Nkv {Nkv}: hot key at {hot}: output != its value row"


@pytest.mark.parametrize("hd", (64, 40))
@pytest.mark.parametrize("Nkv2", (1, 4, 64))
def test_ip_multi_tile(Nkv2, hd):
    """The IP variant over text segments of two and four 128-column tiles: s = 0 equals the plain kernel bit for bit.
    The image segment holds at most 64 tokens, so the doubled-segment identity (image tokens = text tokens, s = 1
    equals the plain kernel on 2·v) runs on the first Nkv2 text tokens as both segments."""
    from cfgpp_b200 import _native as nv
    B, H, Nq, hdp = 2, 2, 200, padded(hd)
    g = gen(hd * 7 + Nkv2)

    def run(q, k, v, k2, v2, s):
        return nv.op_attention_ip(q, k, v, k2, v2, torch.tensor([s], dtype=torch.float32, device=dev), H, head_dim=hd)

    for Nkv in (200, 500):
        q, k, v = (heads(t, hdp) for t in family("peaked", g, B, Nq, Nkv, H, hd))
        k, v = fused(k, v)
        k2, v2 = fused(*(heads(t, hdp) for t in family("flat", g, B, 1, Nkv2, H, hd)[1:]))
        plain = nv.op_attention(q, k, v, H, head_dim=hd)
        assert torch.equal(run(q, k, v, k2, v2, 0.0), plain), f"hd{hd} {Nq}x{Nkv}+{Nkv2}: s = 0 != plain"
        ks, vs = k[:, :Nkv2].contiguous(), v[:, :Nkv2].contiguous()
        assert torch.equal(run(q, ks, vs, ks, vs, 1.0), nv.op_attention(q, ks, vs * 2, H, head_dim=hd)), \
            f"hd{hd} {Nq}x{Nkv2}+{Nkv2}: doubled segment"
