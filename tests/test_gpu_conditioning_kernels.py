"""Kernel-level tests of the small kernels of the ControlNet conditioning embedding and the CLIP vision tower, through
their op-level entry points: `clip_patchify_kernel` and `clip_vision_embed_kernel` (`text_kernels.cu`),
`image_to_nhwc_kernel` and `silu_kernel` (`elementwise.cu`). Each is a copy, one rounding or one fp32 function, so the
answers are bit-exact against torch: unfold / permute with +0 padding, `.half()` of the fp32 sum, the correctly rounded
SiLU (away from rounding ties).

Then the two executors against chains of their per-element pinned ops, bit for bit: `NativeControlNet.embed` equals
image_to_nhwc → (conv3x3 → SiLU)* → conv_out with the weights zero-padded in torch to the packed layout (pinning
`packed_conv3x3`, the strides, the padded widths and where SiLU runs), and `NativeCLIPVisionEncoder.encode` equals
patchify → patch GEMM → vision_embed → pre-LN → per layer (LN, qkv over heads padded in torch, attention, out_proj +
residual, LN, fc1, activation, fc2 + residual) → class row → post-LN → projection."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


def pad64(c):
    return -(-c // 64) * 64


def bits(t):
    return t.contiguous().view(torch.int16)


def assert_bits(what, got, want):
    neq = bits(got) != bits(want)
    n = int(neq.sum())
    if n:
        i = neq.reshape(-1).nonzero()[0].item()
        raise AssertionError(f"{what}: {n} elements differ, first flat index {i}: got {got.reshape(-1)[i].item()}, "
                             f"want {want.reshape(-1)[i].item()}")
    print(f"[conditioning kernels] {what}: bit-exact ({got.numel()} elements)")


def fp32_edges():
    """fp32 values at fp16's rounding edges: ties (1 + 2^-11, 2049, -3073), just past ties, the overflow threshold
    (65504, 65519.99, the tie 65520 and beyond, to ±inf), subnormals and the tie below the smallest one (2^-25)."""
    v = [1 + 2 ** -11, 1 + 3 * 2 ** -11, 2049.0, -3073.0, 2049.0001, 65504.0, 65519.99, 65520.0, -65520.0, 70000.0,
         -1e6, 2 ** -24, 2 ** -25, 3 * 2 ** -26, -2 ** -25, 5e-6, -6.1e-5, 6.0e-8, 1e-9, 0.0, -0.0]
    return torch.tensor(v, dtype=torch.float32)


def plant(x, vals, g):
    """x with `vals` written at random positions (a copy)."""
    x = x.clone().reshape(-1)
    idx = torch.randperm(x.numel(), generator=g)[:vals.numel()]
    x[idx] = vals.to(x.dtype)
    return x


# ---- patchify -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("S,P", [(224, 14), (32, 8)])
def test_clip_patchify(S, P, dtype):
    """Patch rows in (c, ky, kx) column order against unfold, columns K..Kp−1 exactly +0 (Kp = 640 > K = 588 at 224/14;
    Kp = K = 192 at 32/8); fp32 inputs at fp16 ties, past 65504 and in the subnormal range round as `.half()` does."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(S + P)
    B, K = 3, 3 * P * P
    Kp = pad64(K)
    x = torch.randn(B, 3, S, S, generator=g) * 3
    x = plant(x, fp32_edges().repeat(20), g).reshape(B, 3, S, S)
    x = x.to(dtype).to(dev)
    got = nv.op_clip_patchify(x, P, Kp)
    want = torch.zeros(B * (S // P) ** 2, Kp, dtype=torch.float16, device=dev)
    want[:, :K] = F.unfold(x.float(), P, stride=P).transpose(1, 2).reshape(-1, K).half()
    assert_bits(f"patchify {S}/{P} {str(dtype)[6:]} Kp {Kp}", got, want)


# ---- vision embeddings ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("D", [320, 1280, 1664])
@pytest.mark.parametrize("B", [1, 3, 16])
def test_clip_vision_embed(B, D):
    """fp16(cat(cls, pe) + pos) with one rounding, 257 tokens; some sums overflow to ±inf."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(B * 10 + D)
    np_, T = 256, 257
    pe = torch.randn(B * np_, D, generator=g)
    pe = plant(pe, torch.tensor([60000.0, -60000.0, 65504.0, 2 ** -24] * 8), g).reshape(B * np_, D).half().to(dev)
    cls = torch.randn(D, generator=g).half().to(dev)
    cls[:4] = torch.tensor([65504.0, -65504.0, 2 ** -24, -2 ** -24])
    pos = torch.randn(T, D, generator=g)
    pos[1:, :8] = 30000.0
    pos[0, :4] = torch.tensor([40.0, -40.0, 2 ** -24, 2 ** -24])
    pos = pos.half().to(dev)
    got = nv.op_clip_vision_embed(pe, cls, pos, B)
    want = (torch.cat([cls.expand(B, 1, D), pe.view(B, np_, D)], 1).float() + pos.float()).half().reshape(B * T, D)
    assert torch.isinf(want).any(), "no sum overflows"
    assert_bits(f"vision_embed B{B} D{D}", got, want)


# ---- image in -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("B,H,W", [(1, 64, 48), (3, 17, 13), (2, 512, 512), (8, 1024, 1024)])
def test_image_to_nhwc(B, H, W, dtype):
    """The control image [B, 3, H, W] to NHWC with channels 3..63 exactly +0, fp32 rounded as `.half()` does."""
    from cfgpp_b200 import _native as nv
    g = torch.Generator().manual_seed(B * H + W)
    x = torch.rand(B, 3, H, W, generator=g)
    x = plant(x, fp32_edges().repeat(10), g).reshape(B, 3, H, W).to(dtype).to(dev)
    got = nv.op_image_to_nhwc(x, 64)
    want = torch.zeros(B, H, W, 64, dtype=torch.float16, device=dev)
    want[..., :3] = x.permute(0, 2, 3, 1).half()
    assert_bits(f"image_to_nhwc {B}x{H}x{W} {str(dtype)[6:]}", got, want)


# ---- SiLU -----------------------------------------------------------------------------------------------------------

def ulp16(y):
    _, e = torch.frexp(y.abs())
    return torch.ldexp(torch.ones_like(y), e - 11).clamp_min(2.0 ** -24)


def test_silu_every_fp16_input():
    """All 65536 fp16 bit patterns. Every finite output lies within 1 ulp of fp64 silu and equals the correctly rounded
    value except where fp64 silu lies within 2^-20 (relative) of a rounding tie; ±0, ±inf and NaN behave as F.silu."""
    from cfgpp_b200 import _native as nv
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16).to(dev)
    got = nv.op_silu(x.clone())
    torch_silu = F.silu(x)
    exact = F.silu(x.double())
    fin = torch.isfinite(x) & torch.isfinite(exact)
    g, e = got[fin].double(), exact[fin]
    assert torch.isfinite(got[fin]).all(), "finite input, non-finite output"
    err = ((g - e).abs() / ulp16(e)).max().item()
    u = ulp16(e)
    frac = (e.abs() / u) % 1.0
    near_tie = (frac - 0.5).abs() * u <= 2.0 ** -20 * e.abs()
    cr = e.half()
    wrong = (bits(got[fin]) != bits(cr)) & ~near_tie
    special = ~torch.isfinite(x) | (x == 0)
    same_special = (bits(got[special]) == bits(torch_silu[special])) | (torch.isnan(got[special]) &
                                                                        torch.isnan(torch_silu[special]))
    diff_torch = int((bits(got) != bits(torch_silu)).sum())
    print(f"[conditioning kernels] silu: max {err:.3f} ulp of fp64, {int(near_tie.sum())} inputs near a tie, "
          f"{int(wrong.sum())} not correctly rounded elsewhere, {diff_torch} differ from F.silu on the device")
    assert err <= 1.0
    assert not wrong.any(), f"not correctly rounded at x = {x[fin][wrong][:8].tolist()}"
    assert same_special.all(), f"special inputs differ from F.silu: {x[special][~same_special].tolist()}"


# ---- composition: the ControlNet conditioning embedding -------------------------------------------------------------

def embed_chain(cn_cfg, sd, image):
    """The conditioning embedding from the pinned ops, weights zero-padded in torch as `packed_conv3x3` lays them
    out ([Cout_p][tap][Cin_p], bias padded with zeros)."""
    from cfgpp_b200 import _native as nv
    ch = cn_cfg.conditioning_embedding_out_channels
    C0 = cn_cfg.unet.block_out_channels[0]
    e = "controlnet_cond_embedding."

    def conv(x, name, cout_p, stride, silu):
        w, b = sd[e + name + ".weight"].half(), sd[e + name + ".bias"].half()
        cout, cin = w.shape[:2]
        cin_p = x.shape[3]
        wp = torch.zeros(cout_p, 9, cin_p, dtype=torch.float16, device=dev)
        wp[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, 9, cin)
        bp = torch.zeros(cout_p, dtype=torch.float16, device=dev)
        bp[:cout] = b
        y = nv.op_conv3x3_ex(x.contiguous(), wp.reshape(cout_p, 9 * cin_p), bp, stride=stride, pad=1)
        return nv.op_silu(y) if silu else y

    x = nv.op_image_to_nhwc(image, pad64(cn_cfg.conditioning_channels))
    x = conv(x, "conv_in", pad64(ch[0]), 1, True)
    for i in range(len(ch) - 1):
        x = conv(x, f"blocks.{2 * i}", pad64(ch[i]), 1, True)
        x = conv(x, f"blocks.{2 * i + 1}", pad64(ch[i + 1]), 2, True)
    return conv(x, "conv_out", C0, 1, False)


@pytest.mark.parametrize("model,B,S", [("sd15", 2, 512), ("sdxl", 1, 1024)])
def test_conditioning_embedding_equals_its_ops(model, B, S):
    from cfgpp_b200 import config as C, controlnet as CN
    cn_cfg = CN.controlnet_config(C.CONFIGS[model]())
    sd = CN.synthetic_controlnet_state_dict(cn_cfg, seed=3, device=dev)
    cn = CN.NativeControlNet(cn_cfg, sd, dev)
    try:
        image = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(S)).to(dev)
        got = cn.embed(image)
    finally:
        cn.close()
    want = embed_chain(cn_cfg, sd, image)
    assert_bits(f"{model} conditioning embedding B{B} {S}x{S} vs its ops", got, want)


# ---- composition: the CLIP vision tower -----------------------------------------------------------------------------

def vision_chain(cfg, sd, px):
    """image_embeds from the pinned ops, in `ClipVisionEncoder::encode` / `build_clip_layers` order."""
    from cfgpp_b200 import _native as nv
    D, I, H, P, S = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.patch_size, cfg.image_size
    hd = D // H
    hdp = pad64(hd)
    Cp, K, B, T, eps = H * hdp, 3 * P * P, px.shape[0], cfg.num_positions, cfg.layer_norm_eps
    act = {"quick_gelu": 0, "gelu": 1}[cfg.hidden_act]
    vm = "vision_model."

    def w(k):
        return sd[k].half()

    patches = nv.op_clip_patchify(px, P, pad64(K))
    wp = torch.zeros(D, pad64(K), dtype=torch.float16, device=dev)
    wp[:, :K] = w(vm + "embeddings.patch_embedding.weight").reshape(D, K)
    pe = nv.op_linear(patches, wp)
    emb = nv.op_clip_vision_embed(pe, w(vm + "embeddings.class_embedding"),
                                  w(vm + "embeddings.position_embedding.weight"), B)
    x0 = nv.op_layernorm(emb, w(vm + "pre_layrnorm.weight"), w(vm + "pre_layrnorm.bias"), eps)
    for l in range(cfg.num_hidden_layers):
        p = f"{vm}encoder.layers.{l}."
        wqkv = torch.zeros(3, H, hdp, D, dtype=torch.float16, device=dev)
        bqkv = torch.zeros(3, H, hdp, dtype=torch.float16, device=dev)
        for i, n in enumerate(("q_proj", "k_proj", "v_proj")):
            wqkv[i, :, :hd] = w(p + f"self_attn.{n}.weight").view(H, hd, D)
            bqkv[i, :, :hd] = w(p + f"self_attn.{n}.bias").view(H, hd)
        wo = torch.zeros(D, H, hdp, dtype=torch.float16, device=dev)
        wo[:, :, :hd] = w(p + "self_attn.out_proj.weight").view(D, H, hd)
        ln = nv.op_layernorm(x0, w(p + "layer_norm1.weight"), w(p + "layer_norm1.bias"), eps)
        qkv = nv.op_linear(ln, wqkv.reshape(3 * Cp, D), bqkv.reshape(-1)).view(B, T, 3 * Cp)
        att = nv.op_attention(qkv[:, :, :Cp], qkv[:, :, Cp:2 * Cp], qkv[:, :, 2 * Cp:], H, head_dim=hd)
        x1 = nv.op_linear(att.view(B * T, Cp), wo.reshape(D, Cp), w(p + "self_attn.out_proj.bias"), addend=x0)
        ln = nv.op_layernorm(x1, w(p + "layer_norm2.weight"), w(p + "layer_norm2.bias"), eps)
        m = nv.op_clip_activation(nv.op_linear(ln, w(p + "mlp.fc1.weight"), w(p + "mlp.fc1.bias")), act)
        x0 = nv.op_linear(m, w(p + "mlp.fc2.weight"), w(p + "mlp.fc2.bias"), addend=x1)
    cls = x0.view(B, T, D)[:, 0].contiguous()
    cls = nv.op_layernorm(cls, w(vm + "post_layernorm.weight"), w(vm + "post_layernorm.bias"), eps)
    out, _ = nv.op_small_linear(cls, w("visual_projection.weight"))
    return out


@pytest.mark.parametrize("tower,B", [("tiny_vision", 1), ("tiny_vision", 3), ("vit_h", 2), ("vit_bigg", 1)])
def test_vision_tower_equals_its_ops(tower, B):
    from cfgpp_b200 import vision_encoder as V
    cfg = getattr(V, f"{tower}_config")()
    sd = V.synthetic_state_dict(cfg, seed=3, device=dev)
    enc = V.NativeCLIPVisionEncoder(cfg, sd, dev)
    try:
        px = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(B)).to(dev)
        got = enc.encode(px)
    finally:
        enc.close()
    want = vision_chain(cfg, sd, px)
    assert_bits(f"{tower} B{B} image_embeds vs its ops", got, want)
