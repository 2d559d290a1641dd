"""The UNet and AutoencoderKL executors against chains of their pinned ops, bit for bit.

Every kernel the executors launch is pinned element by element against fp64 elsewhere (the GEMM and its epilogues,
the 3x3 convolution in every mode, flash attention, GroupNorm / LayerNorm, the small UNet / VAE kernels). What those
pins cannot see is how `Unet::build` and `VaeDecoder::prepare` wire the kernels together: the skip stack, each
resnet's rows of the one concatenated `time_emb_proj`, the two-source GroupNorm and shortcut of the up blocks, the
LayerNorm fold and its three statistics slots, head padding, GEGLU row packing, the epsilons, the in-place residual /
ControlNet / T2I adds and the decoupled IP attention. A wrong epsilon or a resnet reading its neighbour's temb rows
changes every image by a few ulp and passes a rel-L2 tolerance; here it fails.

`unet_chain` computes (eps_uc, eps_c) the way `Unet::build` / `run_inputs` / `run_body` / `unet_forward` do, in plan
order, calling only the `_native` op wrappers; torch only moves data, to lay weights out as the weight store packs
them. It records the plan-step name of every op it runs, and the list must equal `NativeUNet.profile_forward`'s, so a
plan step added or removed without a counterpart here fails too. `vae_decode_chain` / `vae_encode_chain` do the same
for `VaeDecoder::prepare` / `prepare_encode` (bit equality only: those plans have no names)."""
import numpy as np
import pytest
import torch

import production as P

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


def pad64(c):
    return -(-c // 64) * 64


# ---- comparison -----------------------------------------------------------------------------------------------------

def _ordered(t):
    """fp16 / fp32 bit patterns as integers ordered like the values, so that a difference counts ulp."""
    if t.dtype == torch.float16:
        b, m = t.contiguous().view(torch.int16).long(), 0x7FFF
    else:
        b, m = t.contiguous().view(torch.int32).long(), 0x7FFFFFFF
    return torch.where(b < 0, -(b & m), b)


def assert_bits(what, got, want):
    assert got.dtype == want.dtype and got.shape == want.shape, f"{what}: {got.dtype}{tuple(got.shape)} vs " \
                                                                f"{want.dtype}{tuple(want.shape)}"
    a, b = _ordered(got), _ordered(want)
    neq = a != b
    n = int(neq.sum())
    if n:
        ulp = int((a - b).abs().max())
        raise AssertionError(f"{what}: {n} of {got.numel()} elements differ, by up to {ulp} ulp")


# ---- weight layouts of the weight store (data movement only) --------------------------------------------------------

def conv_packed(w):
    """(Cout, Cin, 3, 3) -> [Cout][tap][Cin] (`packed_conv3x3`)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


def heads_rows(ws, heads, hd, hdp):
    """Stacked (heads*hd, K) projections -> [(mat, head, hdp)][K], rows hd..hdp-1 of every head zero."""
    K = ws[0].shape[1]
    out = torch.zeros(len(ws), heads, hdp, K, dtype=torch.float16, device=dev)
    for i, w in enumerate(ws):
        out[i, :, :hd] = w.view(heads, hd, K)
    return out.reshape(-1, K)


def heads_cols(w, heads, hd, hdp):
    """(N, heads*hd) -> (N, heads*hdp), columns hd..hdp-1 of every head zero."""
    N = w.shape[0]
    out = torch.zeros(N, heads, hdp, dtype=torch.float16, device=dev)
    out[:, :, :hd] = w.view(N, heads, hd)
    return out.reshape(N, -1)


def geglu_packed(w):
    """GEGLU proj rows (2*inner[, K]): every 256 packed rows hold 128 value rows, then the 128 matching gate rows."""
    inner = w.shape[0] // 2
    return w.reshape(2, inner // 128, 128, -1).transpose(0, 1).reshape(w.shape).contiguous()


# ---- the UNet -------------------------------------------------------------------------------------------------------

class UNetChain:
    """One UNet (or the ControlNet, `prefix` "controlnet:") as a chain of op wrappers. `names` collects the plan-step
    names of the per-step forward, in launch order."""

    def __init__(self, cfg, sd, B, H, W, names, prefix="", is_cn=False):
        from cfgpp_b200 import _native as nv
        self.nv, self.cfg, self.sd, self.names, self.prefix, self.is_cn = nv, cfg, sd, names, prefix, is_cn
        self.B, self.NB, self.H, self.W = B, 2 * B, H, W
        self.L, self.boc = len(cfg.block_out_channels), cfg.block_out_channels
        self.t2i = None  # (features, on-word tensor)
        self.ip = None  # (image tokens [NB * T, D], T, scale tensor)
        self._t2i_k = 0
        # resnet order = temb column offsets: down blocks, mid block, then (not a ControlNet) up blocks
        self.temb_off, off, keys = {}, 0, []
        L, lpb = self.L, cfg.layers_per_block
        order = [(f"down_blocks.{i}.resnets.{j}", self.boc[i]) for i in range(L) for j in range(lpb)]
        order += [("mid_block.resnets.0", self.boc[-1]), ("mid_block.resnets.1", self.boc[-1])]
        if not is_cn:
            order += [(f"up_blocks.{i}.resnets.{j}", self.boc[L - 1 - i]) for i in range(L) for j in range(lpb + 1)]
        for p, c in order:
            self.temb_off[p] = off
            off += c
            keys.append(p)
        self.temb_w = torch.cat([self.w(p + ".time_emb_proj.weight") for p in keys])
        self.temb_b = torch.cat([self.w(p + ".time_emb_proj.bias") for p in keys])

    def w(self, key):
        return self.sd[key].to(dev, torch.float16)

    def wlin(self, key):
        """A linear or 1x1-conv weight as [N, K]."""
        t = self.w(key)
        return t.reshape(t.shape[0], -1)

    def step(self, name, out):
        self.names.append(self.prefix + name)
        return out

    # -- prompt-time work (cfgpp_set_prompt): not part of the per-step plan --
    def prompt(self, ctx, pooled=None, time_ids=None):
        nv, cfg = self.nv, self.cfg
        self.ctx = ctx.reshape(-1, cfg.cross_attention_dim)
        self.aug = None
        if cfg.addition_embed_type == "text_time":
            NB, PD, ATE, NT = self.NB, cfg.pooled_dim, cfg.addition_time_embed_dim, cfg.num_time_ids
            AIN = cfg.projection_class_embeddings_input_dim
            add_in = torch.empty(NB, AIN, dtype=torch.float16, device=dev)
            nv.op_copy_rows(pooled, add_in, NB)  # rows r <- r % add_rows, as set_prompt broadcasts them
            tids = time_ids.float().repeat(NB // time_ids.shape[0], 1).reshape(-1).contiguous()
            for j in range(NT):  # one sinusoid per time id, at its column offset
                nv.op_timestep_embedding(tids[j:], NB, ATE, out=add_in, val_stride=NT, col_off=PD + j * ATE)
            h1, _ = nv.op_small_linear(add_in, self.w("add_embedding.linear_1.weight"),
                                       self.w("add_embedding.linear_1.bias"), out_silu=True)
            self.aug, _ = nv.op_small_linear(h1, self.w("add_embedding.linear_2.weight"),
                                             self.w("add_embedding.linear_2.bias"))

    # -- prologue: timestep embedding -> every resnet's time_emb_proj --
    def prologue(self, t):
        nv, C0 = self.nv, self.boc[0]
        tt = torch.tensor([t], dtype=torch.float32, device=dev)
        t_sin = self.step("time_proj", nv.op_timestep_embedding(tt, 1, C0))
        t_h1, _ = self.step("time_embedding.linear_1+silu", nv.op_small_linear(
            t_sin, self.w("time_embedding.linear_1.weight"), self.w("time_embedding.linear_1.bias"), out_silu=True))
        _, semb = self.step("time_embedding.linear_2(+aug_emb)", nv.op_small_linear(
            t_h1, self.w("time_embedding.linear_2.weight"), self.w("time_embedding.linear_2.bias"), addend=self.aug,
            rows=self.NB, want_out2=True))
        self.temb, _ = self.step("resnets.time_emb_proj", nv.op_small_linear(semb, self.temb_w, self.temb_b))

    def conv_in(self, z, in_scale, cond=None):
        nv, C0 = self.nv, self.boc[0]
        s = torch.tensor([in_scale], dtype=torch.float32, device=dev)
        w, b = self.w("conv_in.weight").reshape(C0, 36), self.w("conv_in.bias")
        if cond is None:
            return self.step("conv_in", nv.op_conv_in(z, w, b, s, reps=2))
        return self.step("conv_in(+cond)", nv.op_conv_in_add(z, w, b, cond, s, reps=2))

    # -- blocks --
    def resnet(self, p, x1, x2=None):
        nv, NB, eps = self.nv, self.NB, self.cfg.norm_eps
        _, H, W, C1 = x1.shape
        C2 = 0 if x2 is None else x2.shape[3]
        Cin, Cout, HW = C1 + C2, self.w(p + ".conv1.bias").shape[0], H * W
        x1v, x2v = x1.view(NB, HW, C1), None if x2 is None else x2.view(NB, HW, C2)
        n = self.step(p + ".norm1+silu", nv.op_groupnorm(x1v, self.w(p + ".norm1.weight"), self.w(p + ".norm1.bias"),
                                                        eps, True, x2=x2v))
        off = self.temb_off[p]
        h1 = self.step(p + ".conv1", nv.op_conv3x3_ex(n.view(NB, H, W, Cin), conv_packed(self.w(p + ".conv1.weight")),
                                                     self.w(p + ".conv1.bias"), addend=self.temb[:, off:off + Cout],
                                                     add_rows_per_group=HW))
        n = self.step(p + ".norm2+silu", nv.op_groupnorm(h1.view(NB, HW, Cout), self.w(p + ".norm2.weight"),
                                                        self.w(p + ".norm2.bias"), eps, True))
        res = x1.view(-1, C1)
        if Cin != Cout:
            res = self.step(p + ".conv_shortcut", nv.op_linear(
                x1.view(-1, C1), self.wlin(p + ".conv_shortcut.weight"), self.w(p + ".conv_shortcut.bias"),
                a2=None if x2 is None else x2.view(-1, C2)))
        return self.step(p + ".conv2", nv.op_conv3x3_ex(n.view(NB, H, W, Cout), conv_packed(self.w(p + ".conv2.weight")),
                                                        self.w(p + ".conv2.bias"), addend=res))

    def transformer(self, p, x, layers, heads):
        nv, NB = self.nv, self.NB
        _, H, W, C = x.shape
        HW, Mi = H * W, NB * H * W
        hd = C // heads
        hdp = pad64(hd)
        Cp = heads * hdp

        def producer(name, a, wt, bias, addend=None, out=None):
            # the default tile width, or the widest of 160 / 128 / 64 that tiles C (every column feeds the statistics)
            bn = nv.linear_schedule(a, wt, bias, addend=addend, out=out)["bn"]
            if C % bn:
                bn = next(b for b in (160, 128, 64) if C % b == 0)
            return self.step(name, nv.op_linear_stats(a, wt, bn, bias, addend=addend, out=out))

        def consumer(name, wt, bias, norm, stats, geglu=False):
            wf, s, t = nv.op_fold_ln(wt, self.w(norm + ".weight"), self.w(norm + ".bias"), bias)
            return self.step(name, nv.op_linear_lnfold(tok, wf, s, t, stats, eps=1e-5, geglu=geglu))

        n = self.step(p + ".norm", nv.op_groupnorm(x.view(NB, HW, C), self.w(p + ".norm.weight"),
                                                  self.w(p + ".norm.bias"), 1e-6, False))
        tok, st = producer(p + ".proj_in", n.view(Mi, C), self.wlin(p + ".proj_in.weight"), self.w(p + ".proj_in.bias"))
        for k in range(layers):
            b = f"{p}.transformer_blocks.{k}"
            wqkv = heads_rows([self.w(f"{b}.attn1.to_{m}.weight") for m in "qkv"], heads, hd, hdp)
            qkv = consumer(b + ".attn1.to_qkv(+norm1)", wqkv, None, b + ".norm1", st).view(NB, HW, 3 * Cp)
            a = self.step(b + ".attn1.sdpa", nv.op_attention(qkv[:, :, :Cp], qkv[:, :, Cp:2 * Cp], qkv[:, :, 2 * Cp:],
                                                             heads, head_dim=hd))
            _, st = producer(b + ".attn1.to_out", a.view(Mi, Cp),
                             heads_cols(self.w(b + ".attn1.to_out.0.weight"), heads, hd, hdp),
                             self.w(b + ".attn1.to_out.0.bias"), addend=tok, out=tok)
            wq = heads_rows([self.w(b + ".attn2.to_q.weight")], heads, hd, hdp)
            q = consumer(b + ".attn2.to_q(+norm2)", wq, None, b + ".norm2", st).view(NB, HW, Cp)
            # cross-attention K / V: projected once per prompt
            wkv = heads_rows([self.w(b + ".attn2.to_k.weight"), self.w(b + ".attn2.to_v.weight")], heads, hd, hdp)
            kv = nv.op_linear(self.ctx, wkv).view(NB, -1, 2 * Cp)
            if self.ip is not None:  # the image tokens' K / V, once per image
                tokens, T, scale = self.ip
                pk = self.ip_w[b + ".attn2.processor.to_k_ip.0.weight"]
                pv = self.ip_w[b + ".attn2.processor.to_v_ip.0.weight"]
                kvi = nv.op_linear(tokens, heads_rows([pk, pv], heads, hd, hdp)).view(NB, T, 2 * Cp)
                a = nv.op_attention_ip(q, kv[:, :, :Cp], kv[:, :, Cp:], kvi[:, :, :Cp], kvi[:, :, Cp:], scale, heads,
                                       head_dim=hd)
            else:
                a = nv.op_attention(q, kv[:, :, :Cp], kv[:, :, Cp:], heads, head_dim=hd)
            self.step(b + ".attn2.sdpa", a)
            _, st = producer(b + ".attn2.to_out", a.view(Mi, Cp),
                             heads_cols(self.w(b + ".attn2.to_out.0.weight"), heads, hd, hdp),
                             self.w(b + ".attn2.to_out.0.bias"), addend=tok, out=tok)
            ff = consumer(b + ".ff.geglu(+norm3)", geglu_packed(self.w(b + ".ff.net.0.proj.weight")),
                          geglu_packed(self.w(b + ".ff.net.0.proj.bias")), b + ".norm3", st, geglu=True)
            _, st = producer(b + ".ff.out", ff, self.w(b + ".ff.net.2.weight"), self.w(b + ".ff.net.2.bias"),
                             addend=tok, out=tok)
        out = nv.op_linear(tok, self.wlin(p + ".proj_out.weight"), self.w(p + ".proj_out.bias"), addend=x.view(Mi, C))
        return self.step(p + ".proj_out", out.view(NB, H, W, C))

    def downsample(self, p, x):
        return self.step(p + ".conv", self.nv.op_conv3x3_ex(x, conv_packed(self.w(p + ".conv.weight")),
                                                            self.w(p + ".conv.bias"), stride=2))

    def upsample(self, p, x):
        up = self.step(p + ".nearest2x", self.nv.op_upsample2x(x))
        return self.step(p + ".conv", self.nv.op_conv3x3_ex(up, conv_packed(self.w(p + ".conv.weight")),
                                                            self.w(p + ".conv.bias")))

    def t2i_add(self, h):
        """In place on a down-path output (`add_t2i_feature`), gated by the device word."""
        if self.t2i is None or self._t2i_k >= len(self.t2i[0]):
            return
        from ctypes import c_int, c_size_t
        feats, word = self.t2i
        k = self._t2i_k
        self._t2i_k += 1
        nv = self.nv
        per = h[0].numel()
        nv.check(nv.load().cfgpp_op_t2i_add(nv.ptr(h), nv.ptr(feats[k]), c_int(self.NB), c_int(self.B),
                                            c_size_t(per), nv.ptr(word), nv.stream_ptr()))
        self.step(f"t2i_adapter.add{k}", h)

    # -- the plans --
    def down_mid(self, h0):
        """Down path and mid block; returns the residual list (every skip, then the mid-block output)."""
        cfg, L = self.cfg, self.L
        h = h0
        skips = [h]
        for i in range(L):
            attn = cfg.down_block_types[i] == "CrossAttnDownBlock2D"
            for j in range(cfg.layers_per_block):
                h = self.resnet(f"down_blocks.{i}.resnets.{j}", h)
                if attn:
                    h = self.transformer(f"down_blocks.{i}.attentions.{j}", h, cfg.transformer_layers_per_block[i],
                                         cfg.num_attention_heads[i])
                    if j == cfg.layers_per_block - 1:
                        self.t2i_add(h)
                skips.append(h)
            if i != L - 1:
                h = self.downsample(f"down_blocks.{i}.downsamplers.0", h)
                skips.append(h)
            if not attn:
                self.t2i_add(h)
        h = self.resnet("mid_block.resnets.0", h)
        h = self.transformer("mid_block.attentions.0", h, cfg.transformer_layers_per_block[-1],
                             cfg.num_attention_heads[-1])
        h = self.resnet("mid_block.resnets.1", h)
        self.t2i_add(h)
        return skips + [h]

    def up_tail(self, res):
        cfg, L, nv = self.cfg, self.L, self.nv
        skips, h = res[:-1], res[-1]
        for i in range(L):
            for j in range(cfg.layers_per_block + 1):
                h = self.resnet(f"up_blocks.{i}.resnets.{j}", h, skips.pop())
                if cfg.up_block_types[i] == "CrossAttnUpBlock2D":
                    h = self.transformer(f"up_blocks.{i}.attentions.{j}", h, cfg.transformer_layers_per_block[L - 1 - i],
                                         cfg.num_attention_heads[L - 1 - i])
            if i != L - 1:
                h = self.upsample(f"up_blocks.{i}.upsamplers.0", h)
        assert not skips
        NB, H, W, C0 = h.shape
        n = self.step("conv_norm_out+silu", nv.op_groupnorm(h.view(NB, H * W, C0), self.w("conv_norm_out.weight"),
                                                            self.w("conv_norm_out.bias"), cfg.norm_eps, True))
        wo = self.w("conv_out.weight").permute(0, 2, 3, 1).reshape(4, 9, C0).contiguous()
        eu, ec, _ = self.step("conv_out+step", nv.op_conv_out_step(n.view(NB, H, W, C0), wo, self.w("conv_out.bias")))
        return eu, ec


def unet_chain(cfg, sd, z, t, in_scale, ctx, pooled=None, time_ids=None, cn=None, t2i=None, ip=None):
    """(eps_uc, eps_c, plan names) of one forward. cn = (cn_cfg, cn_sd, cond [B,h,w,C0], scale);
    t2i = (features, on); ip = (adapter weights, image tokens [NB * T, D], T, scale)."""
    from cfgpp_b200 import _native as nv
    B, _, H, W = z.shape
    names = []
    u = UNetChain(cfg, sd, B, H, W, names)
    if t2i is not None:
        u.t2i = ([f.contiguous() for f in t2i[0]], torch.tensor([1 if t2i[1] else 0], dtype=torch.int32, device=dev))
    if ip is not None:
        u.ip_w = {k: v.to(dev, torch.float16) for k, v in ip[0].items()}
        u.ip = (ip[1], ip[2], torch.tensor([ip[3]], dtype=torch.float32, device=dev))
    u.prompt(ctx, pooled, time_ids)
    c = None
    if cn is not None:
        c = UNetChain(cn[0].unet, cn[1], B, H, W, names, prefix="controlnet:", is_cn=True)
        c.prompt(ctx, pooled, time_ids)
    u.prologue(t)
    if c is not None:
        c.prologue(t)
    h0 = u.conv_in(z, in_scale)
    if c is not None:
        cres = c.down_mid(c.conv_in(z, in_scale, cond=cn[2]))
    res = u.down_mid(h0)
    if c is not None:  # the zero convs: scaled and added in place into the skips and the mid-block output
        scale = torch.tensor([cn[3]], dtype=torch.float32, device=dev)
        keys = [f"controlnet_down_blocks.{k}" for k in range(len(res) - 1)] + ["controlnet_mid_block"]
        for k, key in enumerate(keys):
            C = res[k].shape[3]
            r = res[k].view(-1, C)
            u.step(key, nv.op_linear_scaled_residual(cres[k].view(-1, C), c.wlin(key + ".weight"), r, scale,
                                                     c.w(key + ".bias"), out=r))
    eu, ec = u.up_tail(res)
    return eu, ec, names


# ---- cases ----------------------------------------------------------------------------------------------------------

_NET = {}


def _unet(name):
    """(cfg, state dict, NativeUNet) of a config, one at a time: the full-size models do not all fit at once."""
    from cfgpp_b200 import config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    if name not in _NET:
        _release()
        cfg = C.CONFIGS[name]()
        sd = Wt.synthetic_state_dict(cfg, seed=1234, device=dev)
        _NET[name] = (cfg, sd, NativeUNet(cfg, sd, dev))
    return _NET[name]


def _release():
    for _, _, net in _NET.values():
        net.close()
    _NET.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _close_nets():
    yield
    _release()


def _inputs(cfg, B, h, w, seed, zdtype, add_rows):
    """Seeded inputs with distinct rows: latents, per-row prompts, pooled embeddings and time ids."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 4, h, w, generator=g).to(zdtype).to(dev)
    ctx = torch.randn(2 * B, P.N_CTX, cfg.cross_attention_dim, generator=g).half().to(dev)
    pooled = tids = None
    if cfg.addition_embed_type == "text_time":
        rows = 2 * B if add_rows == "2B" else B
        pooled = torch.randn(rows, cfg.pooled_dim, generator=g).half().to(dev)
        base = [8 * h, 8 * w, 0, 0, 8 * h, 8 * w, 6.0][:cfg.num_time_ids]
        tids = torch.tensor([[v + 13 * r + 3 * k for k, v in enumerate(base)] for r in range(rows)],
                            dtype=torch.float32, device=dev)
    return z, ctx, pooled, tids


C_IN = 1.0 / (14.6 ** 2 + 1) ** 0.5  # k-diffusion's c_in at sigma_max


def _run(name, B, h, w, t, in_scale=1.0, zdtype=torch.float32, add_rows="2B", seed=7, cn=None, t2i=None, ip=None):
    """predict_noise and profile_forward of the native handle against unet_chain. `cn` = (cn_cfg, cn_sd, native
    ControlNet, scale); `t2i` = on; `ip` = (IPAdapter, scale)."""
    from cfgpp_b200 import t2i_adapter as T
    from cfgpp_b200 import _native as nv
    cfg, sd, net = _unet(name)
    z, ctx, pooled, tids = _inputs(cfg, B, h, w, seed, zdtype, add_rows)
    g = torch.Generator().manual_seed(seed + 1)
    chain_cn = chain_t2i = chain_ip = None
    try:
        net.attach_controlnet(None if cn is None else cn[2])
        net.attach_ip_adapter(None if ip is None else ip[0])
        feats = None
        if t2i is not None:
            feats = [(torch.randn(B, hh, ww, c, generator=g) * 0.5).half().to(dev)
                     for c, hh, ww in T.unet_placements(cfg, h, w)]
        net.attach_t2i(0 if feats is None else len(feats))
        net.prepare(B, h, w)
        net.set_prompt(ctx, pooled, tids)
        if cn is not None:
            image = torch.rand(B, 3, 8 * h, 8 * w, generator=g).to(dev)
            net.set_control_image(image)
            net.set_control_scale(cn[3])
            chain_cn = (cn[0], cn[1], cn[2].embed(image), cn[3])
        if feats is not None:
            net.set_t2i_features(feats)
            net.set_t2i_active(t2i)
            chain_t2i = (feats, t2i)
        if ip is not None:
            ad, scale = ip
            if ad.resampler is not None:
                e = (torch.randn(B, ad.resampler["seq_len"], ad.embed_dim, generator=g)).half().to(dev)
            else:
                e = torch.randn(B, ad.embed_dim, generator=g).half().to(dev)
            net.set_ip_image_embeds(e)
            net.set_ip_adapter_scale(scale)
            if ad.resampler is not None:  # the Resampler over the rows the engine hands it, unconditional rows first
                from test_gpu_encoder_chains import resampler_chain
                tokens = resampler_chain(ad.weights, ad.image_rows(e), ad.resampler, cfg.cross_attention_dim)
            else:  # image_proj: Linear(E -> T * D), then LayerNorm(D) of every token
                rows = torch.cat([torch.zeros_like(e), e])
                D, Tn = cfg.cross_attention_dim, ad.n_tokens
                wp = ad.weights
                proj = nv.op_linear(rows, wp["image_proj.proj.weight"].to(dev, torch.float16),
                                    wp["image_proj.proj.bias"].to(dev, torch.float16))
                tokens = nv.op_layernorm(proj.view(2 * B * Tn, D), wp["image_proj.norm.weight"].to(dev, torch.float16),
                                         wp["image_proj.norm.bias"].to(dev, torch.float16), 1e-5)
            chain_ip = (ad.weights, tokens, ad.n_tokens, scale)
        eu, ec = net.predict_noise(z, t, in_scale)
        plan = [n for n, _, _, _ in net.profile_forward(z, t, in_scale)]
        again = net.predict_noise(z, t, in_scale)
    finally:
        net.attach_controlnet(None)
        net.attach_ip_adapter(None)
        net.attach_t2i(0)
    assert torch.equal(eu, again[0]) and torch.equal(ec, again[1]), "predict_noise is not deterministic"
    ceu, cec, names = unet_chain(cfg, sd, z, t, in_scale, ctx, pooled, tids, cn=chain_cn, t2i=chain_t2i, ip=chain_ip)
    torch.cuda.synchronize()
    assert names == plan, _plan_diff(plan, names)
    what = f"{name} B{B} {h}x{w} t={t} in_scale={in_scale:.5g} z {str(zdtype)[6:]}"
    assert_bits(what + " eps_uc", eu, ceu)
    assert_bits(what + " eps_c", ec, cec)
    print(f"[executor chains] {what}: {len(plan)} plan steps, eps bit-exact")


def _plan_diff(plan, names):
    for i, (a, b) in enumerate(zip(plan, names)):
        if a != b:
            return f"plan step {i}: executor {a!r}, chain {b!r}"
    return f"executor has {len(plan)} steps, chain {len(names)}: first extra " \
           f"{(plan if len(plan) > len(names) else names)[min(len(plan), len(names))]!r}"


@pytest.mark.parametrize("name,h,w", P.unet_sizes(), ids=[P.size_tag(*s) for s in P.unet_sizes()])
def test_unet_production_size_equals_its_ops(name, h, w):
    """Every full-size UNet at every production latent, batch 1 (SD v1.5 is the config with padded heads)."""
    _run(name, 1, h, w, 500.37)


@pytest.mark.parametrize("name,B,hw,t,in_scale,zdtype,add_rows", [
    ("tiny_sd15", 3, 32, 1.0, 1.0, torch.float16, "2B"),
    ("tiny_sd2", 3, 32, 500.37, C_IN, torch.float32, "2B"),
    ("tiny_sdxl", 3, 32, 999.0, C_IN, torch.float16, "2B"),
    ("tiny_sdxl", 3, 32, 500.37, 1.0, torch.float32, "B"),
    ("tiny_sdxl_refiner", 2, 32, 1.0, C_IN, torch.float32, "B"),
    ("sdxl", 2, 128, 999.0, C_IN, torch.float16, "2B"),
], ids=["sd15-b3-f16z", "sd2-b3-cin", "sdxl-b3-cin-f16z", "sdxl-b3-undup", "refiner-b2-undup", "sdxl128-b2"])
def test_unet_per_image_rows_equal_its_ops(name, B, hw, t, in_scale, zdtype, add_rows):
    """Distinct prompts, pooled embeddings and time ids per row, so every image has its own temb rows; fp32 and fp16
    latents, in_scale 1 and a k-diffusion c_in, integral and fractional t; SDXL with and without duplicated rows."""
    _run(name, B, hw, hw, t, in_scale, zdtype, add_rows)


def _controlnet(name):
    from cfgpp_b200 import config as C, controlnet as CN
    cn_cfg = CN.controlnet_config(C.CONFIGS[name]())
    cn_sd = CN.synthetic_controlnet_state_dict(cn_cfg, seed=4321, device=dev)
    return cn_cfg, cn_sd, CN.NativeControlNet(cn_cfg, cn_sd, dev)


@pytest.mark.parametrize("name,B,hw", [("tiny_sd15", 2, 32), ("tiny_sdxl", 1, 32), ("sdxl", 1, 128)])
def test_controlnet_equals_its_ops(name, B, hw):
    """The ControlNet's down path and mid block (conv_in plus the embedded control image), then the zero convs added
    in place into the skips at scale 0.7."""
    cfg, sd, net = _unet(name)
    cn_cfg, cn_sd, cn = _controlnet(name)
    try:
        _run(name, B, hw, hw, 500.37, C_IN, cn=(cn_cfg, cn_sd, cn, 0.7))
    finally:
        cn.close()


@pytest.mark.parametrize("name,B,hw,on", [("tiny_sdxl", 2, 32, True), ("tiny_sd15", 1, 32, True),
                                          ("tiny_sd15", 2, 32, False), ("sd15", 1, 64, True)])
def test_t2i_adapter_equals_its_ops(name, B, hw, on):
    """The features added in place at every placement, with the device word on and off."""
    _run(name, B, hw, hw, 999.0, 1.0, t2i=on)


@pytest.mark.parametrize("name,B,hw,plus", [("tiny_sd15", 2, 32, False), ("tiny_sdxl", 1, 32, True),
                                            ("sd15", 1, 64, False), ("sdxl", 1, 128, True)])
def test_ip_adapter_equals_its_ops(name, B, hw, plus):
    """The decoupled cross-attention over the image tokens at scale 0.6: image_proj (Linear + LayerNorm) for the
    plain adapter, `resampler_chain` over the hidden-state rows for Plus, then every block's to_k_ip / to_v_ip."""
    from cfgpp_b200 import ip_adapter as IP
    cfg, _, _ = _unet(name)
    ad = IP.IPAdapter(f"chain-{name}", dev, cfg, image_proj="resampler" if plus else None)
    try:
        _run(name, B, hw, hw, 500.37, 1.0, ip=(ad, 0.6))
    finally:
        ad.close()


# ---- the AutoencoderKL ----------------------------------------------------------------------------------------------

class VaeChain:
    def __init__(self, sd):
        from cfgpp_b200 import _native as nv
        self.nv, self.sd = nv, sd

    def w(self, key):
        return self.sd[key].to(dev, torch.float16)

    def resnet(self, p, x, Cout):
        nv = self.nv
        B, H, W, Cin = x.shape
        n = nv.op_groupnorm(x.view(B, H * W, Cin), self.w(p + ".norm1.weight"), self.w(p + ".norm1.bias"), 1e-6, True)
        h1 = nv.op_conv3x3_ex(n.view(B, H, W, Cin), conv_packed(self.w(p + ".conv1.weight")), self.w(p + ".conv1.bias"))
        n = nv.op_groupnorm(h1.view(B, H * W, Cout), self.w(p + ".norm2.weight"), self.w(p + ".norm2.bias"), 1e-6, True)
        res = x.view(-1, Cin)
        if Cin != Cout:
            res = nv.op_linear(res, self.w(p + ".conv_shortcut.weight").reshape(Cout, Cin),
                               self.w(p + ".conv_shortcut.bias"))
        return nv.op_conv3x3_ex(n.view(B, H, W, Cout), conv_packed(self.w(p + ".conv2.weight")),
                                self.w(p + ".conv2.bias"), addend=res)

    def attention(self, p, x):
        """One head of width C over all H*W tokens: S = Q Kᵀ per image, row softmax, Vᵀ = W_v Xᵀ, P Vᵀ + b_v."""
        nv = self.nv
        B, H, W, C = x.shape
        N = H * W
        n = nv.op_groupnorm(x.view(B, N, C), self.w(p + ".group_norm.weight"), self.w(p + ".group_norm.bias"), 1e-6,
                            False).view(B * N, C)
        q = nv.op_linear(n, self.w(p + ".to_q.weight"), self.w(p + ".to_q.bias"))
        k = nv.op_linear(n, self.w(p + ".to_k.weight"), self.w(p + ".to_k.bias"))
        # 1 / sqrtf(C) in fp32; the op, like the executor, multiplies it by log2(e) in fp32
        scale = float(np.float32(1.0) / np.sqrt(np.float32(C)))
        o = torch.empty(B * N, C, dtype=torch.float16, device=dev)
        for s in range(B):
            r = slice(s * N, (s + 1) * N)
            sc = nv.op_vae_row_softmax(nv.op_linear(q[r], k[r]), scale)
            vt = nv.op_linear(self.w(p + ".to_v.weight"), n[r])
            nv.op_linear(sc, vt, self.w(p + ".to_v.bias"), out=o[r])
        out = nv.op_linear(o, self.w(p + ".to_out.0.weight"), self.w(p + ".to_out.0.bias"), addend=x.view(B * N, C))
        return out.view(B, H, W, C)


def vae_decode_chain(cfg, sd, z):
    """`VaeDecoder::prepare`'s plan: latent prep, conv_in, mid block, up blocks, GroupNorm + SiLU, conv to RGB."""
    v = VaeChain(sd)
    nv, boc, L = v.nv, cfg.block_out_channels, len(cfg.block_out_channels)
    Ct = boc[-1]
    zq = nv.op_vae_latent_prep(z, cfg.scaling_factor, v.w("post_quant_conv.weight").reshape(4, 4),
                               v.w("post_quant_conv.bias"))
    x = nv.op_conv_in(zq, v.w("decoder.conv_in.weight").reshape(Ct, 36), v.w("decoder.conv_in.bias"))
    x = v.resnet("decoder.mid_block.resnets.0", x, Ct)
    x = v.attention("decoder.mid_block.attentions.0", x)
    x = v.resnet("decoder.mid_block.resnets.1", x, Ct)
    for i in range(L):
        blk = f"decoder.up_blocks.{i}"
        for j in range(cfg.layers_per_block + 1):
            x = v.resnet(f"{blk}.resnets.{j}", x, boc[L - 1 - i])
        if i != L - 1:
            x = nv.op_conv3x3_ex(nv.op_upsample2x(x), conv_packed(v.w(blk + ".upsamplers.0.conv.weight")),
                                 v.w(blk + ".upsamplers.0.conv.bias"))
    B, H, W, C = x.shape
    n = nv.op_groupnorm(x.view(B, H * W, C), v.w("decoder.conv_norm_out.weight"), v.w("decoder.conv_norm_out.bias"),
                        1e-6, True)
    wo = v.w("decoder.conv_out.weight").permute(0, 2, 3, 1).reshape(3, 9, C).contiguous()
    return nv.op_vae_conv_rgb(n.view(B, H, W, C), wo, v.w("decoder.conv_out.bias"))


def vae_encode_chain(cfg, sd, x, noise):
    """`VaeDecoder::prepare_encode`'s plan: image pad, conv_in, down blocks with stride-2 pad-0 downsamplers, mid
    block, GroupNorm + SiLU, then conv_out + quant_conv + the posterior sample in one kernel."""
    v = VaeChain(sd)
    nv, boc, L = v.nv, cfg.block_out_channels, len(cfg.block_out_channels)
    C0 = boc[0]
    img4 = nv.op_vae_image_pad(x)
    wci = torch.zeros(C0, 36, dtype=torch.float16, device=dev)  # (C0, 3*9) with the zero plane's 9 columns
    wci[:, :27] = v.w("encoder.conv_in.weight").reshape(C0, 27)
    h = nv.op_conv_in(img4, wci, v.w("encoder.conv_in.bias"))
    for i in range(L):
        blk = f"encoder.down_blocks.{i}"
        for j in range(cfg.layers_per_block):
            h = v.resnet(f"{blk}.resnets.{j}", h, boc[i])
        if i != L - 1:
            h = nv.op_conv3x3_ex(h, conv_packed(v.w(blk + ".downsamplers.0.conv.weight")),
                                 v.w(blk + ".downsamplers.0.conv.bias"), stride=2, pad=0)
    C = boc[-1]
    h = v.resnet("encoder.mid_block.resnets.0", h, C)
    h = v.attention("encoder.mid_block.attentions.0", h)
    h = v.resnet("encoder.mid_block.resnets.1", h, C)
    B, H, W, _ = h.shape
    n = nv.op_groupnorm(h.view(B, H * W, C), v.w("encoder.conv_norm_out.weight"), v.w("encoder.conv_norm_out.bias"),
                        1e-6, True)
    wo = v.w("encoder.conv_out.weight").permute(0, 2, 3, 1).reshape(8, 9, C).contiguous()
    return nv.op_vae_moments_sample(n.view(B, H, W, C), wo, v.w("encoder.conv_out.bias"),
                                    v.w("quant_conv.weight").reshape(8, 8), v.w("quant_conv.bias"), cfg.scaling_factor,
                                    noise)


def _vae_kind(H, W):
    return "sdxl_vae" if H * W >= 1024 * 832 else "sd15_vae"


_VAE_CASES = [(_vae_kind(H, W), 1, H, W) for H, W in P.VAE_SIZES] + [("tiny_vae", 3, 128, 256)]
_VAE_IDS = [f"{k}-b{b}-{W}x{H}" for k, b, H, W in _VAE_CASES]


@pytest.mark.parametrize("kind,B,H,W", _VAE_CASES, ids=_VAE_IDS)
def test_vae_decode_equals_its_ops(kind, B, H, W):
    from cfgpp_b200 import vae as V
    cfg = V.VAE_CONFIGS[kind]()
    sd = V.synthetic_vae_state_dict(cfg, seed=5, device=dev)
    g = torch.Generator().manual_seed(H + W)
    z = (torch.randn(B, 4, H // 8, W // 8, generator=g) * cfg.scaling_factor * 6.0).to(dev)
    dec = V.NativeVAEDecoder(cfg, sd, dev)
    try:
        got = dec.decode_fp16(z)
    finally:
        dec.close()
    want = vae_decode_chain(cfg, sd, z)
    assert_bits(f"vae decode {kind} B{B} {W}x{H}", got, want)


@pytest.mark.parametrize("kind,B,H,W", _VAE_CASES, ids=_VAE_IDS)
def test_vae_encode_equals_its_ops(kind, B, H, W):
    from cfgpp_b200 import vae as V
    cfg = V.VAE_CONFIGS[kind]()
    sd = V.synthetic_vae_state_dict(cfg, seed=9, device=dev, with_encoder=True)
    g = torch.Generator().manual_seed(H * W)
    x = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).half().to(dev)
    noise = torch.randn(B, 4, H // 8, W // 8, generator=g).half().to(dev)
    vae = V.NativeVAEDecoder(cfg, sd, dev)
    try:
        got = vae.encode(x, noise)
    finally:
        vae.close()
    want = vae_encode_chain(cfg, sd, x, noise)
    assert_bits(f"vae encode {kind} B{B} {W}x{H}", got, want)
