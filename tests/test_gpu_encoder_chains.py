"""The executors that feed the UNet against chains of their pinned ops, bit for bit: the CLIP text towers
(`ClipTextEncoder::encode` / `build_clip_layers`), the CLIP vision tower's hidden states (`encode_hidden`, what
IP-Adapter Plus reads), the T2I-Adapter network (`T2IAdapter::prepare`) and the IP-Adapter Plus Resampler
(`Unet::build_ip_resampler`).

Every kernel they launch is pinned element by element elsewhere; the rel-L2 tests against the oracle and transformers
pin the models. What neither sees is the wiring: an epsilon, an fp32 summation order, a scale applied in fp16 or a
wrong row moves every output by a few ulp and still passes a tolerance. Each chain here calls only the `_native` op
wrappers (or the C ABI `cfgpp_op_*` entry points of ops without one), in the executor's order; torch only lays the
weights out as the weight store packs them, slices, repeats and concatenates. Every chain reads its weights through
`Reads`, and each test asserts that the keys read are the model's parameter list, so a chain that skips a weight fails.
The T2I chain also pins its elementwise launches against their exact torch statements on the activations they see
(`t2i_chain`). The cases come from `production.py`, plus tiny configs."""
from ctypes import c_float, c_int, c_size_t
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import production as P
from test_gpu_executor_chains import assert_bits, conv_packed, dev, heads_cols, heads_rows, pad64

pytestmark = pytest.mark.gpu

ENCODE_MAX = 16  # the most prompts / images one native encode takes, and `encode_batch`'s chunk
ACT = {"quick_gelu": 0, "gelu": 1}


class Reads:
    """A state dict that records every key read from it."""

    def __init__(self, sd):
        self.sd, self.keys = sd, set()

    def __getitem__(self, key):
        self.keys.add(key)
        return self.sd[key]


def _half(sd):
    return lambda key: sd[key].to(dev, torch.float16)


_OPEN = {}


def _handle(key, make):
    """One cached (cfg, state dict, native tower) at a time, so that the batches of a tower share one handle."""
    if key not in _OPEN:
        _close_towers()
        _OPEN[key] = make()
    return _OPEN[key]


def _close_towers():
    for *_, h in _OPEN.values():
        h.close()
    _OPEN.clear()


@pytest.fixture(scope="module", autouse=True)
def _close_handles():
    from test_gpu_executor_chains import _release  # the UNets the Resampler cases attach to
    yield
    _close_towers()
    _release()


# ---- the CLIP text towers -------------------------------------------------------------------------------------------

def text_chain(cfg, sd, ids):
    """(hidden_states [L + 1 of [B, T, D]], last_hidden_state [B, T, D], pooled [B, projection_dim or D]) of ids [B, T],
    in `ClipTextEncoder::encode` / `build_clip_layers` order."""
    from cfgpp_b200 import _native as nv, text_encoder as TE
    w = _half(sd)
    B, T = ids.shape
    D, H, eps, act = cfg.hidden_size, cfg.num_attention_heads, cfg.layer_norm_eps, ACT[cfg.hidden_act]
    tm = "text_model."
    ids = ids.to(dev, torch.int32).contiguous()
    x0 = nv.op_clip_embed(ids.view(-1), w(tm + "embeddings.token_embedding.weight"),
                          w(tm + "embeddings.position_embedding.weight")[:T])
    hs = [x0]
    for l in range(cfg.num_hidden_layers):
        p = f"{tm}encoder.layers.{l}."
        a = p + "self_attn."
        # q | k | v as one operand and one bias (64-wide heads: no padding rows)
        wqkv = heads_rows([w(a + f"{m}_proj.weight") for m in "qkv"], H, 64, 64)
        bqkv = heads_rows([w(a + f"{m}_proj.bias")[:, None] for m in "qkv"], H, 64, 64).view(-1)
        ln = nv.op_layernorm(x0, w(p + "layer_norm1.weight"), w(p + "layer_norm1.bias"), eps)
        att = nv.op_clip_attention(nv.op_linear(ln, wqkv, bqkv), B, T, H)
        x1 = nv.op_linear(att, w(a + "out_proj.weight"), w(a + "out_proj.bias"), addend=x0)
        ln = nv.op_layernorm(x1, w(p + "layer_norm2.weight"), w(p + "layer_norm2.bias"), eps)
        m = nv.op_clip_activation(nv.op_linear(ln, w(p + "mlp.fc1.weight"), w(p + "mlp.fc1.bias")), act)
        x0 = nv.op_linear(m, w(p + "mlp.fc2.weight"), w(p + "mlp.fc2.bias"), addend=x1)
        hs.append(x0)
    last = nv.op_layernorm(x0, w(tm + "final_layer_norm.weight"), w(tm + "final_layer_norm.bias"), eps)
    pidx = TE.NativeCLIPTextEncoder.pooled_index(SimpleNamespace(cfg=cfg), ids)
    pooled = nv.op_clip_gather_rows(last, pidx, T)
    if cfg.projection_dim > 0:
        pooled, _ = nv.op_small_linear(pooled, w("text_projection.weight"))
    return [h.view(B, T, D) for h in hs], last.view(B, T, D), pooled


def token_ids(cfg, B, T, seed=3):
    """B rows of T ids: bos, n random tokens, eos, then the tower's pad id (eos for CLIP-L, 0 for bigG and H). n
    cycles through a row without padding (T - 2), the empty prompt (bos then eos), one token, and partial rows."""
    g = torch.Generator().manual_seed(seed)
    bos, eos = cfg.vocab_size - 2, cfg.vocab_size - 1
    ids = torch.full((B, T), cfg.pad_token_id, dtype=torch.int32)
    for b in range(B):
        n = min([T - 2, 0, 1, 5, 23, 40, 11, 60][b % 8], T - 2)
        ids[b, 0] = bos
        ids[b, 1:1 + n] = torch.randint(1, cfg.vocab_size - 3, (n,), generator=g, dtype=torch.int32)
        ids[b, 1 + n] = eos
    return ids


def _text_tower(cfg):
    from cfgpp_b200 import text_encoder as TE

    def make():
        sd = TE.synthetic_clip_state_dict(cfg, seed=21, device=dev)
        return cfg, sd, TE.NativeCLIPTextEncoder(cfg, sd, dev)
    return _handle(cfg, make)


def _check_text(what, enc, cfg, sd, ids):
    """encode at every skip, with every output and with the hidden state alone (the executor then runs L - skip
    layers), and the two conditioner modes without a hidden output, against one chain."""
    from cfgpp_b200 import text_encoder as TE
    reads = Reads(sd)
    hs, last, pooled = text_chain(cfg, reads, ids)
    assert reads.keys == {k for k, _, _ in TE.clip_param_specs(cfg)}, "the chain does not read every weight"
    L = cfg.num_hidden_layers
    for skip in range(L + 1):
        h, la, po = enc.encode(ids, skip=skip)
        assert_bits(f"{what} skip {skip} hidden_states[{L - skip}]", h, hs[L - skip])
        assert_bits(f"{what} skip {skip} last_hidden_state", la, last)
        assert_bits(f"{what} skip {skip} pooled", po, pooled)
        h, _, _ = enc.encode(ids, skip=skip, want_last=False, want_pooled=False)
        assert_bits(f"{what} skip {skip} hidden_states[{L - skip}] alone", h, hs[L - skip])
    _, la, _ = enc.encode(ids, skip=0, want_hidden=False, want_pooled=False)
    assert_bits(f"{what} last_hidden_state alone", la, last)
    _, _, po = enc.encode(ids, skip=1, want_hidden=False, want_last=False)
    assert_bits(f"{what} pooled alone", po, pooled)


_TEXT_CASES = [(t, B) for t, bs in P.TEXT_TOWERS.items() for B in bs] + [("clip_bigg", ENCODE_MAX)]


@pytest.mark.parametrize("tower,B", _TEXT_CASES, ids=[f"{t}-b{B}" for t, B in _TEXT_CASES])
def test_text_tower_equals_its_ops(tower, B):
    """Every production tower at its prompt batches, and bigG at the encode maximum: 77 tokens, rows padded with the
    tower's pad id, a row without padding, the empty prompt and a one-token prompt."""
    from cfgpp_b200 import text_encoder as TE
    cfg, sd, enc = _text_tower(TE.CLIP_CONFIGS[tower]())
    T = cfg.max_position_embeddings
    _check_text(f"{tower} B{B}", enc, cfg, sd, token_ids(cfg, B, T, seed=B))


_TINY_TEXT = [(act, proj, T) for act in ACT for proj in (0, 64) for T in (77, 13)]


@pytest.mark.parametrize("act,proj,T", _TINY_TEXT, ids=[f"tiny-{a}-proj{p}-t{T}" for a, p, T in _TINY_TEXT])
def test_tiny_text_tower_equals_its_ops(act, proj, T):
    """quick_gelu and gelu, with and without a text projection, at 77 tokens and at 13 (fewer than max_positions:
    the position table is read at rows 0..12)."""
    from cfgpp_b200 import text_encoder as TE
    cfg, sd, enc = _text_tower(TE.tiny_clip_config(proj, act))
    _check_text(f"tiny {act} proj {proj} T{T}", enc, cfg, sd, token_ids(cfg, 5, T, seed=T))


def test_text_plan_reuse_equals_its_ops():
    """One handle encodes at batch 8, then 1, then 8 (each a new plan); every result equals the chain and a fresh
    handle."""
    from cfgpp_b200 import text_encoder as TE
    cfg, sd, enc = _text_tower(TE.clip_bigg_config())
    T = cfg.max_position_embeddings
    for i, B in enumerate((8, 1, 8)):
        ids = token_ids(cfg, B, T, seed=40 + i)
        got = enc.encode(ids)
        hs, last, pooled = text_chain(cfg, sd, ids)
        fresh = TE.NativeCLIPTextEncoder(cfg, sd, dev)
        try:
            again = fresh.encode(ids)
        finally:
            fresh.close()
        for what, a, b, c in zip(("hidden", "last", "pooled"), got, (hs[-2], last, pooled), again):
            assert_bits(f"bigG encode {i} B{B} {what} vs its ops", a, b)
            assert_bits(f"bigG encode {i} B{B} {what} vs a fresh handle", a, c)


# ---- the CLIP vision tower ------------------------------------------------------------------------------------------

def vision_chain(cfg, sd, px):
    """(image_embeds [B, projection_dim], hidden_states [L + 1 of [B, T, D]]) from the pinned ops, in
    `ClipVisionEncoder::embed` / `encode` / `build_clip_layers` order, heads padded in torch to whole 64-wide blocks."""
    from cfgpp_b200 import _native as nv
    w = _half(sd)
    D, H, Pz = cfg.hidden_size, cfg.num_attention_heads, cfg.patch_size
    hd = D // H
    hdp = pad64(hd)
    Cp, K, B, T, eps = H * hdp, 3 * Pz * Pz, px.shape[0], cfg.num_positions, cfg.layer_norm_eps
    act = ACT[cfg.hidden_act]
    vm = "vision_model."
    patches = nv.op_clip_patchify(px, Pz, pad64(K))
    pe = nv.op_linear(patches, heads_cols(w(vm + "embeddings.patch_embedding.weight").reshape(D, K), 1, K, pad64(K)))
    emb = nv.op_clip_vision_embed(pe, w(vm + "embeddings.class_embedding"),
                                  w(vm + "embeddings.position_embedding.weight"), B)
    x0 = nv.op_layernorm(emb, w(vm + "pre_layrnorm.weight"), w(vm + "pre_layrnorm.bias"), eps)
    hs = [x0]
    for l in range(cfg.num_hidden_layers):
        p = f"{vm}encoder.layers.{l}."
        a = p + "self_attn."
        wqkv = heads_rows([w(a + f"{m}_proj.weight") for m in "qkv"], H, hd, hdp)
        bqkv = heads_rows([w(a + f"{m}_proj.bias")[:, None] for m in "qkv"], H, hd, hdp).view(-1)
        ln = nv.op_layernorm(x0, w(p + "layer_norm1.weight"), w(p + "layer_norm1.bias"), eps)
        qkv = nv.op_linear(ln, wqkv, bqkv).view(B, T, 3 * Cp)
        att = nv.op_attention(qkv[:, :, :Cp], qkv[:, :, Cp:2 * Cp], qkv[:, :, 2 * Cp:], H, head_dim=hd)
        x1 = nv.op_linear(att.view(B * T, Cp), heads_cols(w(a + "out_proj.weight"), H, hd, hdp),
                          w(a + "out_proj.bias"), addend=x0)
        ln = nv.op_layernorm(x1, w(p + "layer_norm2.weight"), w(p + "layer_norm2.bias"), eps)
        m = nv.op_clip_activation(nv.op_linear(ln, w(p + "mlp.fc1.weight"), w(p + "mlp.fc1.bias")), act)
        x0 = nv.op_linear(m, w(p + "mlp.fc2.weight"), w(p + "mlp.fc2.bias"), addend=x1)
        hs.append(x0)
    cls = x0.view(B, T, D)[:, 0].contiguous()
    cls = nv.op_layernorm(cls, w(vm + "post_layernorm.weight"), w(vm + "post_layernorm.bias"), eps)
    out, _ = nv.op_small_linear(cls, w("visual_projection.weight"))
    return out, [h.view(B, T, D) for h in hs]


def _vision_chain_split(cfg, sd, px):
    """vision_chain over the slices of at most ENCODE_MAX images that `encode` / `encode_hidden` hand the library."""
    parts = [vision_chain(cfg, sd, px[i:i + ENCODE_MAX]) for i in range(0, px.shape[0], ENCODE_MAX)]
    return torch.cat([e for e, _ in parts]), [torch.cat(h) for h in zip(*[hs for _, hs in parts])]


def _vision_cases():
    out = [("tiny_vision", B, dt, "all") for B, dt in ((1, "f32"), (3, "f32"), (3, "f16"), (ENCODE_MAX + 1, "f32"))]
    out += [("vit_h", B, "f32", 1) for B in P.VISION_TOWERS["vit_h"]] + [("vit_h", P.VISION_TOWERS["vit_h"][0], "f16", 1)]
    return out + [("vit_bigg", 1, "f32", 1)]


_DT = {"f32": torch.float32, "f16": torch.float16}


@pytest.mark.parametrize("tower,B,dtype,skips", _vision_cases(),
                         ids=[f"{t}-b{B}-{d}-skip{s}" for t, B, d, s in _vision_cases()])
def test_vision_hidden_states_equal_its_ops(tower, B, dtype, skips):
    """encode_hidden at every skip of the tiny tower (B = 17 is split at 16 in Python), ViT-H at its production batches
    and ViT-bigG at skip 1 (the Plus path), fp32 and fp16 pixels; encode's image_embeds on the same chain."""
    from cfgpp_b200 import vision_encoder as V
    cfg = P.vision_config(tower)

    def make():
        sd = V.synthetic_state_dict(cfg, seed=3, device=dev)
        return cfg, sd, V.NativeCLIPVisionEncoder(cfg, sd, dev)
    _, sd, enc = _handle(tower, make)
    g = torch.Generator().manual_seed(B)
    px = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=g).to(dev, _DT[dtype])
    reads = Reads(sd)
    embeds, hs = _vision_chain_split(cfg, reads, px)
    assert reads.keys == {k for k, _, _ in V.param_specs(cfg)}, "the chain does not read every weight"
    L = cfg.num_hidden_layers
    for skip in range(L + 1) if skips == "all" else (skips,):
        assert_bits(f"{tower} B{B} {dtype} hidden_states[{L - skip}]", enc.encode_hidden(px, skip=skip), hs[L - skip])
    assert_bits(f"{tower} B{B} {dtype} image_embeds", enc.encode(px), embeds)


_PLUS_BASES = ["tiny_sd15"] + [m for m, _ in P.IP_PLUS_ADAPTERS]


@pytest.mark.parametrize("name", _PLUS_BASES)
def test_unconditional_hidden_states_equal_its_ops(name):
    """The Plus adapter's unconditional rows: its tower's penultimate hidden states of the all-zero preprocessed image."""
    from cfgpp_b200 import config as C, ip_adapter as IP
    ad = IP.IPAdapter(f"chain-{name}", dev, C.CONFIGS[name](), image_proj="resampler")
    try:
        sd = ad._enc_sd  # the synthetic tower's weights, released once the tower is built
        got = ad.unconditional_hidden_states()
    finally:
        ad.close()
    S, L = ad.encoder_cfg.image_size, ad.encoder_cfg.num_hidden_layers
    _, hs = vision_chain(ad.encoder_cfg, sd, torch.zeros(1, 3, S, S, device=dev))
    assert_bits(f"{name} Plus unconditional hidden states", got, hs[L - 1])


# ---- the T2I-Adapter ------------------------------------------------------------------------------------------------

def t2i_chain(cfg, sd, image, scale):
    """The features of `T2IAdapter::prepare`'s plan: pixel unshuffle, conv_in, then per block the average pool, the
    1x1 in_conv, the resnets (3x3 conv, ReLU, 1x1 conv plus the block input, in place) and the scaled copy.

    The executor and the chain launch the same elementwise kernels, so their equality cannot see inside them; the chain
    therefore also pins each elementwise launch, on the activations it runs on, against its exact torch statement: the
    fp16 rounding of the pixels, the window summed row by row in fp32 from 0 and divided by 4, `x > 0 ? x : 0`, and
    fp16(fp32(x) * scale)."""
    from cfgpp_b200 import _native as nv
    lib, st = nv.load(), nv.stream_ptr()
    w = _half(sd)
    B, Ci, H, W = image.shape
    f = cfg.downscale_factor
    x = torch.empty(B, H // f, W // f, Ci * f * f, dtype=torch.float16, device=dev)
    nv.check(lib.cfgpp_op_pixel_unshuffle(nv.ptr(image), c_int(nv.dtype_code(image)), nv.ptr(x), c_int(B), c_int(Ci),
                                          c_int(H), c_int(W), c_int(f), st))
    assert_bits("pixel unshuffle", x, F.pixel_unshuffle(image.half(), f).permute(0, 2, 3, 1))

    def pool(x, what):
        """The 2x2 average pool launch on x, pinned; returns it and the pairwise-summed mean."""
        _, h, wd, C = x.shape
        y = torch.empty(B, h // 2, wd // 2, C, dtype=torch.float16, device=dev)
        nv.check(lib.cfgpp_op_avgpool2x2(nv.ptr(x), nv.ptr(y), c_int(B), c_int(h), c_int(wd), c_int(C), st))
        v = [x[:, dy::2, dx::2].float() for dy in (0, 1) for dx in (0, 1)]
        assert_bits(f"{what} average pool", y, ((((v[0] + v[1]) + v[2]) + v[3]) / 4).half())
        return y, ((v[0] + v[1]) + (v[2] + v[3])) / 4

    cur = nv.op_conv3x3_ex(x, conv_packed(w("adapter.conv_in.weight")), w("adapter.conv_in.bias"))
    feats = []
    for i, (cin, cout, down) in enumerate(cfg.blocks()):
        p = f"adapter.body.{i}"
        if down:
            y, _ = pool(cur, p)
            # the activations' window sums are nearly always exact in fp32, whatever the order; these planted windows
            # (±1024, 3·2^-16, ∓1024, 2^-14) are not, so that the launch shows its summation order at this shape too
            _, h, wd, C = cur.shape
            planted = cur.clone()
            win = planted.view(B, h // 2, 2, wd // 2, 2, C)[:, ::5]
            sign = (1 - 2 * (torch.arange(C, device=dev) % 2)).half()
            win[:, :, 0, :, 0] = 1024 * sign
            win[:, :, 0, :, 1] = 3 * 2.0 ** -16
            win[:, :, 1, :, 0] = -1024 * sign
            win[:, :, 1, :, 1] = 2.0 ** -14
            yp, pairwise = pool(planted, p + " (planted windows)")
            assert not torch.equal(yp, pairwise.half()), "the planted windows do not depend on the summation order"
            cur = y
        _, h, wd, _ = cur.shape
        M = B * h * wd
        if cin != cout:
            cur = nv.op_linear(cur.view(M, cin), w(p + ".in_conv.weight").reshape(cout, cin),
                               w(p + ".in_conv.bias")).view(B, h, wd, cout)
        for j in range(cfg.num_res_blocks):
            r = f"{p}.resnets.{j}"
            t = nv.op_conv3x3_ex(cur, conv_packed(w(r + ".block1.weight")), w(r + ".block1.bias"))
            relu = torch.where(t > 0, t, torch.zeros_like(t))
            nv.check(lib.cfgpp_op_relu(nv.ptr(t), c_size_t(t.numel()), st))
            assert_bits(f"{r} ReLU", t, relu)
            res = cur.view(M, cout)
            nv.op_linear(t.view(M, cout), w(r + ".block2.weight").reshape(cout, cout), w(r + ".block2.bias"),
                         addend=res, out=res)
        out = torch.empty_like(cur)
        nv.check(lib.cfgpp_op_scale(nv.ptr(cur), c_float(scale), nv.ptr(out), c_size_t(cur.numel()), st))
        assert_bits(f"{p} scale {scale}", out, (cur.float() * scale).half())
        feats.append(out)
    return feats


def _t2i_cases():
    """Every production size x batch x image channels with fp32 images, then one fp16 case per adapter kind."""
    from cfgpp_b200 import config as C, t2i_adapter as T
    out = [(name, h, w, B, Ci, "f32") for name, h, w in P.t2i_sizes() for B in P.T2I_ADAPTER_BATCHES
           for Ci in P.T2I_IN_CHANNELS]
    kinds = {}
    for name, h, w in P.t2i_sizes():
        kinds.setdefault(T.t2i_adapter_config(C.CONFIGS[name]()).adapter_type, (name, h, w))
    return out + [(name, h, w, P.T2I_ADAPTER_BATCHES[-1], 3, "f16") for name, h, w in kinds.values()]


@pytest.mark.parametrize("name,h,w,B,Ci,dtype", _t2i_cases(),
                         ids=[f"{P.size_tag(n, h, w)}-b{B}-c{c}-{d}" for n, h, w, B, c, d in _t2i_cases()])
def test_t2i_adapter_equals_its_ops(name, h, w, B, Ci, dtype):
    """Every feature of NativeT2IAdapter.features at scales 0.8 and 1.0 (full_adapter and full_adapter_xl; SD v1.5 at
    512x768 runs its 96/48/24/12-wide levels through the im2col A tile)."""
    from cfgpp_b200 import config as C, t2i_adapter as T
    cfg = T.t2i_adapter_config(C.CONFIGS[name](), Ci)
    sd = T.synthetic_t2i_adapter_state_dict(cfg, seed=7, device=dev)
    image = torch.rand(B, Ci, 8 * h, 8 * w, generator=torch.Generator().manual_seed(B + h)).to(dev, _DT[dtype])
    ad = T.NativeT2IAdapter(cfg, sd, dev)
    try:
        for scale in (0.8, 1.0):
            got = ad.features(image, scale)
            reads = Reads(sd)
            want = t2i_chain(cfg, reads, image, scale)
            assert reads.keys == {k for k, _, _ in T.t2i_adapter_param_specs(cfg)}, "the chain does not read every weight"
            assert len(got) == len(want)
            for k, (a, b) in enumerate(zip(got, want)):
                assert_bits(f"{P.size_tag(name, h, w)} B{B} C{Ci} {dtype} scale {scale} feature {k}", a, b)
    finally:
        ad.close()


# ---- the IP-Adapter Plus Resampler ----------------------------------------------------------------------------------

def resampler_chain(weights, rows, geometry, D):
    """The image tokens [NB * Q, D] of the hidden-state rows [NB, T, E], in `Unet::build_ip_resampler` order;
    `weights` holds the `image_proj.*` keys, `geometry` is `IPAdapter.resampler`."""
    from cfgpp_b200 import _native as nv
    w = _half(weights)
    NB, T, E = rows.shape
    Q, dim, heads = geometry["num_queries"], geometry["dim"], geometry["heads"]
    inner, S, eps = 64 * heads, T + Q, 1e-5
    p = "image_proj."
    x = nv.op_linear(rows.reshape(NB * T, E), w(p + "proj_in.weight"), w(p + "proj_in.bias"))
    lat = w(p + "latents").reshape(Q, dim).repeat(NB, 1)
    for i in range(geometry["depth"]):
        l = f"{p}layers.{i}."
        kv_in, q_in = nv.op_ip_ln_concat(x.view(NB, T, dim), lat.view(NB, Q, dim), w(l + "0.norm1.weight"),
                                         w(l + "0.norm1.bias"), w(l + "0.norm2.weight"), w(l + "0.norm2.bias"), eps)
        q = nv.op_linear(q_in.view(NB * Q, dim), w(l + "0.to_q.weight")).view(NB, Q, inner)
        kv = nv.op_linear(kv_in.view(NB * S, dim), w(l + "0.to_kv.weight")).view(NB, S, 2 * inner)
        o = nv.op_attention(q, kv[..., :inner], kv[..., inner:], heads, 64)
        lat = nv.op_linear(o.view(NB * Q, inner), w(l + "0.to_out.weight"), addend=lat)
        ln = nv.op_layernorm(lat, w(l + "1.0.weight"), w(l + "1.0.bias"), eps)
        ff = nv.op_clip_activation(nv.op_linear(ln, w(l + "1.1.weight")), 1)
        lat = nv.op_linear(ff, w(l + "1.3.weight"), addend=lat)
    po = nv.op_linear(lat, w(p + "proj_out.weight"), w(p + "proj_out.bias"))
    return nv.op_layernorm(po, w(p + "norm_out.weight"), w(p + "norm_out.bias"), eps)


_RESAMPLER_CASES = [(m, NB // 2) for m, _ in P.IP_PLUS_ADAPTERS for NB in P.IP_PLUS_NB] + \
                   [("tiny_sd15", 3), ("tiny_sdxl", 2)]


@pytest.mark.parametrize("name,B", _RESAMPLER_CASES, ids=[f"{m}-b{B}" for m, B in _RESAMPLER_CASES])
def test_resampler_equals_its_ops(name, B):
    """The Resampler's tokens of B images (UNet batch 2B) as `cfgpp_dbg_ip_image_proj` returns them, from the rows of
    `IPAdapter.image_rows`: the unconditional rows first, as the executor takes them."""
    from cfgpp_b200 import _native as nv, ip_adapter as IP
    from test_gpu_executor_chains import _unet
    cfg, _, net = _unet(name)
    ad = IP.IPAdapter(f"chain-{name}", dev, cfg, image_proj="resampler")
    g = torch.Generator().manual_seed(B)
    hidden = torch.randn(B, ad.resampler["seq_len"], ad.embed_dim, generator=g).half().to(dev)
    try:
        net.attach_ip_adapter(ad)
        net.prepare(B, 32, 32)
        net.set_ip_image_embeds(hidden)
        got = torch.empty(2 * B * ad.n_tokens, cfg.cross_attention_dim, dtype=torch.float16, device=dev)
        nv.check(net.lib.cfgpp_dbg_ip_image_proj(net._h, nv.ptr(got), nv.stream_ptr()))
        rows = ad.image_rows(hidden)
        reads = Reads(ad.weights)
        want = resampler_chain(reads, rows, ad.resampler, cfg.cross_attention_dim)
    finally:
        net.attach_ip_adapter(None)
        ad.close()
    assert reads.keys == {k for k in ad.weights if k.startswith("image_proj.")}, "the chain does not read every weight"
    assert_bits(f"{name} Plus B{B} tokens", got, want)
