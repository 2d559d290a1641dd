"""ctypes binding of libcfgpp_b200.so (the C-ABI boundary declared in include/cfgpp_b200.h).

There is deliberately no fallback: if the library is absent or a call fails, this raises.
PyTorch is used only as the owner of device memory and streams (raw pointers cross the boundary).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_void_p
from pathlib import Path

import torch

# CFGPP_B200_LIB points at an alternative build of the same library (A/B experiments)
_LIB_PATH = Path(os.environ.get("CFGPP_B200_LIB") or Path(__file__).resolve().parent / "lib" / "libcfgpp_b200.so")
_lib = None


class NativeError(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


def load() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise NativeError(
                f"{_LIB_PATH} not found — build it with `python -m cfgpp_b200.build` "
                "(there is no CPU/eager fallback on the product path)")
        _lib = ctypes.CDLL(str(_LIB_PATH))
        _lib.cfgpp_last_error.restype = c_char_p
        _lib.cfgpp_version.restype = c_int
    return _lib


def check(status: int) -> None:
    if status != 0:
        msg = load().cfgpp_last_error()
        raise NativeError(f"cfgpp native call failed ({status}): {msg.decode() if msg else '?'}")


def ptr(t: torch.Tensor | None) -> c_void_p:
    if t is None:
        return c_void_p(0)
    assert t.is_cuda and t.is_contiguous(), "native ops take contiguous CUDA tensors"
    return c_void_p(t.data_ptr())


def rows_ptr(t: torch.Tensor | None) -> c_void_p:
    """A 2-D operand the kernel addresses by rows with its own leading dimension (t.stride(0)): column slices of a
    wider buffer are fine, the columns themselves must be contiguous."""
    if t is None:
        return c_void_p(0)
    assert t.is_cuda and t.dim() == 2 and t.stride(1) == 1, "row-addressed operands need contiguous columns"
    return c_void_p(t.data_ptr())


def stream_ptr() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def dtype_code(t: torch.Tensor) -> int:
    """The C ABI's dtype code of a tensor: 0 fp16, 1 fp32."""
    if t.dtype == torch.float16:
        return 0
    if t.dtype == torch.float32:
        return 1
    raise TypeError(f"unsupported dtype {t.dtype}")


class NativeHandle:
    """Owner of one model handle of the C ABI, whose entry points are cfgpp{_prefix}_create / _load_weight /
    _finalize_weights / _destroy. `_open` creates it on a CUDA device and streams the weights in; `close` (or garbage
    collection) destroys it."""

    _prefix = ""
    _what = ""  # what the handle runs, for the error on a non-CUDA device

    def _entry(self, name: str):
        return getattr(self.lib, f"cfgpp{self._prefix}_{name}")

    def _open(self, desc: ctypes.Structure, weights, device) -> None:
        """Create the handle for `desc` on `device`, load the (key, tensor) pairs of `weights` (fp16 or fp32, any
        device) and finalize."""
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise NativeError(f"the cfgpp_b200 {self._what} runs on CUDA (sm_90a) only; use the oracle for CPU runs")
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", idx)
        self.lib = load()
        self._h = c_void_p()
        with torch.cuda.device(self.device):
            self._create(desc, idx)
            st = stream_ptr()
            for key, w in weights:
                w = w.detach().to(self.device).contiguous()
                shape = (ctypes.c_int64 * w.dim())(*w.shape)
                check(self._entry("load_weight")(self._h, key.encode(), ptr(w), shape, c_int(w.dim()),
                                                 c_int(dtype_code(w)), st))
                del w
            torch.cuda.synchronize(self.device)
            check(self._entry("finalize_weights")(self._h, st))

    def _create(self, desc: ctypes.Structure, idx: int) -> None:
        check(self._entry("create")(ctypes.byref(desc), c_int(idx), ctypes.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            self._entry("destroy")(self._h)
            self._h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


# ------------------------------------------------------------------------------------------------
# operator-level wrappers (one kernel launch each) — used by tests and micro-benchmarks
# ------------------------------------------------------------------------------------------------
def _linear_out(out, M, n_out, device):
    if out is None:
        return torch.empty((M, n_out), dtype=torch.float16, device=device)
    assert out.shape == (M, n_out) and out.dtype == torch.float16 and out.is_contiguous()
    return out


def op_linear(a: torch.Tensor, w: torch.Tensor, bias=None, addend=None, add_rows_per_group: int = 1,
              a2: torch.Tensor | None = None, geglu: bool = False, force_bn: int = 0,
              out: torch.Tensor | None = None, force_streamk: bool = False) -> torch.Tensor:
    """out = epilogue(cat([a, a2], -1) @ w.T); a [M,K1] fp16, w [N,K] fp16 (already packed for GEGLU). `out` may be
    given, also as the residual `addend` itself (in-place residual add). `force_streamk` takes the stream-K remainder
    split that linear layers otherwise skip (tests of its fix-up path). a, a2 and addend may be column slices of wider
    buffers (their row stride is passed as the leading dimension)."""
    lib = load()
    M, K1 = a.shape
    K = K1 + (a2.shape[1] if a2 is not None else 0)
    N = w.shape[0]
    assert w.shape[1] == K and a.dtype == torch.float16 and w.dtype == torch.float16
    n_out = N // 2 if geglu else N
    out = _linear_out(out, M, n_out, a.device)
    check(lib.cfgpp_op_linear(*_linear_args(a, w, bias, addend, add_rows_per_group, a2, geglu, force_bn, ptr(out),
                                            force_streamk), stream_ptr()))
    return out


def _linear_args(a, w, bias, addend, add_rows_per_group, a2, geglu, force_bn, out_ptr, force_streamk):
    M, K1 = a.shape
    N, K = w.shape
    return (rows_ptr(a), c_int(a.stride(0)), rows_ptr(a2), c_int(a2.stride(0) if a2 is not None else 0), c_int(K1),
            ptr(w), c_int(M), c_int(N), c_int(K), ptr(bias), rows_ptr(addend),
            c_int(addend.stride(0) if addend is not None else 0), c_int(add_rows_per_group), out_ptr,
            c_int(N // 2 if geglu else N), c_int(1 if geglu else 0), c_int(force_bn), c_int(1 if force_streamk else 0))


_SCHEDULE_FIELDS = ("bn", "grid", "tiles", "streamk", "sk_tiles", "max_pieces", "a_mode", "k_blocks")
A_MODES = ("linear", "tiled", "im2col")


def _schedule(conv, args):
    info = (c_int * 8)()
    check(load().cfgpp_dbg_gemm_schedule(c_int(conv), *args, info))
    s = dict(zip(_SCHEDULE_FIELDS, info))
    s["streamk"] = bool(s["streamk"])
    s["a_mode"] = A_MODES[s["a_mode"]]
    return s


def linear_schedule(a: torch.Tensor, w: torch.Tensor, bias=None, addend=None, add_rows_per_group: int = 1,
                    a2: torch.Tensor | None = None, geglu: bool = False, force_bn: int = 0,
                    out: torch.Tensor | None = None, force_streamk: bool = False) -> dict:
    """The schedule op_linear would run with these arguments, without launching it (debug entry point): {bn, grid,
    tiles, streamk, sk_tiles, max_pieces, a_mode, k_blocks}. It depends on the card's SM count. Nothing is written:
    without `out`, the output's tensor map is encoded over w's address."""
    args = _linear_args(a, w, bias, addend, add_rows_per_group, a2, geglu, force_bn, ptr(out if out is not None else w),
                        force_streamk)
    return _schedule(0, (*args, c_int(1), c_int(1), c_int(1), c_int(1), c_int(0)))


def conv3x3_schedule(x_nhwc: torch.Tensor, w_packed: torch.Tensor, bias=None, addend=None, add_rows_per_group: int = 1,
                     stride: int = 1, pad: int = 1, force_im2col: bool = False, force_bn: int = 0) -> dict:
    """The schedule op_conv3x3_ex would run with these arguments, without launching it (see linear_schedule; the
    output's tensor map is encoded over x's address)."""
    B, H, W, Cin = x_nhwc.shape
    Cout = w_packed.shape[0]
    return _schedule(1, (ptr(x_nhwc), c_int(Cin), c_void_p(0), c_int(0), c_int(0), ptr(w_packed), c_int(B),
                         c_int(Cout), c_int(9 * Cin), ptr(bias), rows_ptr(addend),
                         c_int(addend.stride(0) if addend is not None else 0), c_int(add_rows_per_group), ptr(x_nhwc),
                         c_int(Cout), c_int(0), c_int(force_bn), c_int(0), c_int(H), c_int(W), c_int(stride), c_int(pad),
                         c_int(1 if force_im2col else 0)))


def op_linear_stats(a: torch.Tensor, w: torch.Tensor, bn: int, bias=None, addend=None, add_rows_per_group: int = 1,
                    out: torch.Tensor | None = None, force_streamk: bool = False):
    """op_linear that also emits the LayerNorm-fold row statistics of its fp16 output (a transformer block's residual
    producer). Returns (out, stats): stats [2 * ceil(N / bn), M, 2] fp32 (sum, sum of squares), part 2 j + h over
    columns [j bn + h bn / 2, j bn + (h + 1) bn / 2)."""
    lib = load()
    M, K = a.shape
    N = w.shape[0]
    assert a.is_contiguous() and w.shape[1] == K and bn > 0
    out = _linear_out(out, M, N, a.device)
    stats = torch.empty((2 * ((N + bn - 1) // bn), M, 2), dtype=torch.float32, device=a.device)
    check(lib.cfgpp_op_linear_lnfold(ptr(a), ptr(w), c_int(M), c_int(N), c_int(K), ptr(bias), ptr(addend),
                                     c_int(addend.stride(0) if addend is not None else 0), c_int(add_rows_per_group),
                                     ptr(out), c_int(N), c_int(0), c_int(bn), c_int(1 if force_streamk else 0),
                                     ptr(stats), c_void_p(0), c_int(0), c_float(0.0), c_void_p(0), c_void_p(0),
                                     stream_ptr()))
    return out, stats


def op_linear_lnfold(h: torch.Tensor, wf: torch.Tensor, s: torch.Tensor, t: torch.Tensor, stats: torch.Tensor,
                     eps: float = 1e-5, geglu: bool = False, force_bn: int = 0, ln_parts: int | None = None,
                     out: torch.Tensor | None = None, force_streamk: bool = False) -> torch.Tensor:
    """LayerNorm(h) @ w.T + bias as the folded GEMM: h [M,C] fp16, (wf, s, t) from op_fold_ln, stats [parts, M, 2]
    fp32 row (sum, sum of squares) partials of h (op_linear_stats, or any split of the columns)."""
    lib = load()
    M, K = h.shape
    N = wf.shape[0]
    parts = stats.shape[0] if ln_parts is None else ln_parts
    assert h.is_contiguous() and wf.shape[1] == K and stats.shape[1:] == (M, 2) and stats.dtype == torch.float32
    assert s.dtype == torch.float32 and t.dtype == torch.float32 and s.shape == t.shape == (N,)
    n_out = N // 2 if geglu else N
    out = _linear_out(out, M, n_out, h.device)
    check(lib.cfgpp_op_linear_lnfold(ptr(h), ptr(wf), c_int(M), c_int(N), c_int(K), c_void_p(0), c_void_p(0), c_int(0),
                                     c_int(1), ptr(out), c_int(n_out), c_int(1 if geglu else 0), c_int(force_bn),
                                     c_int(1 if force_streamk else 0), c_void_p(0), ptr(stats), c_int(parts),
                                     c_float(eps), ptr(s), ptr(t), stream_ptr()))
    return out


def op_linear_scaled_residual(a: torch.Tensor, w: torch.Tensor, addend: torch.Tensor, scale: torch.Tensor | None,
                              bias=None, out: torch.Tensor | None = None, force_bn: int = 0) -> torch.Tensor:
    """The ControlNet zero-conv epilogue: fp16(addend + fp16(fp16(a @ w.T + bias) * s)), s = scale (fp32 [1] device
    tensor; None: the plain residual epilogue). `out` may be `addend` itself (in place)."""
    lib = load()
    M, K = a.shape
    N = w.shape[0]
    assert a.is_contiguous() and w.shape[1] == K and addend.shape == (M, N) and addend.is_contiguous()
    assert scale is None or (scale.dtype == torch.float32 and scale.numel() == 1)
    out = _linear_out(out, M, N, a.device)
    check(lib.cfgpp_op_linear_scaled_residual(ptr(a), ptr(w), c_int(M), c_int(N), c_int(K), ptr(bias), ptr(addend),
                                              ptr(scale), ptr(out), c_int(force_bn), stream_ptr()))
    return out


def op_fold_ln(w: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, bias: torch.Tensor | None = None):
    """The LayerNorm fold of w [N,K] (the production weight preparation): (wf = fp16(w * gamma), s [N] fp32 =
    sum_k wf, t [N] fp32 = w @ beta + bias)."""
    lib = load()
    N, K = w.shape
    wf = torch.empty_like(w)
    s = torch.empty(N, dtype=torch.float32, device=w.device)
    t = torch.empty(N, dtype=torch.float32, device=w.device)
    check(lib.cfgpp_op_fold_ln(ptr(w), ptr(gamma), ptr(beta), ptr(bias), ptr(wf), ptr(s), ptr(t), c_int(N), c_int(K),
                               stream_ptr()))
    return wf, s, t


def op_lora_merge(base: torch.Tensor, downs, ups, coefs, out: torch.Tensor | None = None) -> torch.Tensor:
    """The LoRA merge kernel: fp16(fp32(base) + sum_a coefs[a] * ups[a] @ downs[a]) with fp32 accumulation and one
    rounding; base [N,K] fp16, downs[a] [r_a,K], ups[a] [N,r_a] fp16, up to 4 adapters of rank 1..128."""
    lib = load()
    N, K = base.shape
    n = len(downs)
    assert len(ups) == n and len(coefs) == n and base.dtype == torch.float16
    for d, u in zip(downs, ups):
        assert d.dtype == u.dtype == torch.float16 and d.shape == (u.shape[1], K) and u.shape[0] == N
    out = torch.empty_like(base) if out is None else out
    check(lib.cfgpp_op_lora_merge(ptr(base), (c_void_p * n)(*[d.data_ptr() for d in downs]),
                                  (c_void_p * n)(*[u.data_ptr() for u in ups]),
                                  (c_int * n)(*[d.shape[0] for d in downs]), (c_float * n)(*[float(c) for c in coefs]),
                                  c_int(n), c_int(N), c_int(K), ptr(out), stream_ptr()))
    return out


def op_conv3x3(x_nhwc: torch.Tensor, w_packed: torch.Tensor, bias=None, addend=None,
               add_rows_per_group: int = 1, force_bn: int = 0) -> torch.Tensor:
    """x [B,H,W,Cin] fp16 NHWC, w_packed [Cout, 9*Cin] (tap-major), returns [B,H,W,Cout]."""
    lib = load()
    B, H, W, Cin = x_nhwc.shape
    Cout = w_packed.shape[0]
    assert w_packed.shape[1] == 9 * Cin
    out = torch.empty((B, H, W, Cout), dtype=torch.float16, device=x_nhwc.device)
    check(lib.cfgpp_op_conv3x3(ptr(x_nhwc), c_int(B), c_int(H), c_int(W), c_int(Cin), ptr(w_packed), c_int(Cout),
                               ptr(bias), ptr(addend), c_int(addend.stride(0) if addend is not None else 0),
                               c_int(add_rows_per_group), ptr(out), c_int(force_bn), stream_ptr()))
    return out


def op_conv3x3_s2(x_nhwc: torch.Tensor, w_packed: torch.Tensor, bias=None, pad: int = 1) -> torch.Tensor:
    """Downsample2D conv: x [B,H,W,Cin] fp16 NHWC (even H, W), w_packed [Cout, 9*Cin] (tap-major) -> [B,H/2,W/2,Cout].
    pad=1: symmetric zero padding (UNet); pad=0: one zero row / column after the image (AutoencoderKL encoder)."""
    lib = load()
    B, H, W, Cin = x_nhwc.shape
    Cout = w_packed.shape[0]
    out = torch.empty((B, H // 2, W // 2, Cout), dtype=torch.float16, device=x_nhwc.device)
    check(lib.cfgpp_op_conv3x3_s2(ptr(x_nhwc), c_int(B), c_int(H), c_int(W), c_int(Cin), ptr(w_packed), c_int(Cout),
                                  ptr(bias), c_int(pad), ptr(out), stream_ptr()))
    return out


def op_conv3x3_ex(x_nhwc: torch.Tensor, w_packed: torch.Tensor, bias=None, addend=None, add_rows_per_group: int = 1,
                  stride: int = 1, pad: int = 1, force_im2col: bool = False, force_bn: int = 0) -> torch.Tensor:
    """The 3x3 convolution in every mode: x [B,H,W,Cin] fp16 NHWC, w_packed [Cout, 9*Cin] (tap-major) ->
    [B,H/stride,W/stride,Cout]; stride 1 / pad 1, stride 2 / pad 1 (Downsample2D) or stride 2 / pad 0 (one zero row /
    column after the image). Any H, W: the A tile comes through the im2col tensor map where the tiled box cannot hold
    128 consecutive output pixels; `force_im2col` takes the im2col map everywhere (mode comparisons)."""
    lib = load()
    B, H, W, Cin = x_nhwc.shape
    Cout = w_packed.shape[0]
    assert w_packed.shape[1] == 9 * Cin
    out = torch.empty((B, H // stride, W // stride, Cout), dtype=torch.float16, device=x_nhwc.device)
    check(lib.cfgpp_op_conv3x3_ex(ptr(x_nhwc), c_int(B), c_int(H), c_int(W), c_int(Cin), ptr(w_packed), c_int(Cout),
                                  ptr(bias), rows_ptr(addend), c_int(addend.stride(0) if addend is not None else 0),
                                  c_int(add_rows_per_group), ptr(out), c_int(force_bn), c_int(stride), c_int(pad),
                                  c_int(1 if force_im2col else 0), stream_ptr()))
    return out


def op_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, head_dim: int = 64) -> torch.Tensor:
    """q [B,Nq,H*P], k/v [B,Nkv,H*P] fp16 (views with a row stride are fine) -> [B,Nq,H*P]; P = head_dim rounded up
    to a multiple of 64, the padding columns of every head being zero."""
    lib = load()
    B, Nq, C = q.shape
    Nkv = k.shape[1]
    out = torch.empty((B, Nq, C), dtype=torch.float16, device=q.device)
    for t in (q, k, v):
        assert t.is_cuda and t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
    check(lib.cfgpp_op_attention(c_void_p(q.data_ptr()), c_int(q.stride(1)), c_void_p(k.data_ptr()), c_int(k.stride(1)),
                                 c_void_p(v.data_ptr()), c_int(v.stride(1)), ptr(out), c_int(C), c_int(B),
                                 c_int(heads), c_int(Nq), c_int(Nkv), c_int(head_dim), stream_ptr()))
    return out


def op_attention_ip(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, k2: torch.Tensor, v2: torch.Tensor,
                    scale: torch.Tensor, heads: int, head_dim: int = 64) -> torch.Tensor:
    """Decoupled cross-attention: op_attention over (k, v) plus s times a softmax attention over the image tokens
    k2 / v2 [B,Nkv2,H*P] (Nkv2 <= 64), summed in fp32 and rounded once; s = scale[0], an fp32 device tensor the kernel
    reads (a view into a larger tensor is fine)."""
    lib = load()
    B, Nq, C = q.shape
    Nkv, Nkv2 = k.shape[1], k2.shape[1]
    out = torch.empty((B, Nq, C), dtype=torch.float16, device=q.device)
    for t in (q, k, v, k2, v2):
        assert t.is_cuda and t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
    assert scale.is_cuda and scale.dtype == torch.float32
    check(lib.cfgpp_op_attention_ip(c_void_p(q.data_ptr()), c_int(q.stride(1)), c_void_p(k.data_ptr()),
                                    c_int(k.stride(1)), c_void_p(v.data_ptr()), c_int(v.stride(1)),
                                    c_void_p(k2.data_ptr()), c_int(k2.stride(1)), c_void_p(v2.data_ptr()),
                                    c_int(v2.stride(1)), c_int(Nkv2), c_void_p(scale.data_ptr()), ptr(out), c_int(C),
                                    c_int(B), c_int(heads), c_int(Nq), c_int(Nkv), c_int(head_dim), stream_ptr()))
    return out


def op_groupnorm(x1: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, silu: bool,
                 x2: torch.Tensor | None = None) -> torch.Tensor:
    """x1 [B,HW,C1] (+ x2 [B,HW,C2]) NHWC fp16 -> GroupNorm(32) over the channel concat, optional SiLU."""
    lib = load()
    B, HW, C1 = x1.shape
    C2 = x2.shape[2] if x2 is not None else 0
    out = torch.empty((B, HW, C1 + C2), dtype=torch.float16, device=x1.device)
    check(lib.cfgpp_op_groupnorm(ptr(x1), c_int(C1), ptr(x2), c_int(C2), c_int(B), c_int(HW), ptr(gamma), ptr(beta),
                                 c_float(eps), c_int(1 if silu else 0), ptr(out), stream_ptr()))
    return out


def op_layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    lib = load()
    M, C = x.shape
    out = torch.empty_like(x)
    check(lib.cfgpp_op_layernorm(ptr(x), c_int(M), c_int(C), ptr(gamma), ptr(beta), c_float(eps), ptr(out),
                                 stream_ptr()))
    return out


def op_ip_ln_concat(x: torch.Tensor, lat: torch.Tensor, g0: torch.Tensor, b0: torch.Tensor, g1: torch.Tensor,
                    b1: torch.Tensor, eps: float = 1e-5):
    """The two LayerNorms of a Resampler layer in one launch: x [NB, T, C], lat [NB, Q, C] fp16 ->
    (kv [NB, T + Q, C] = cat(LN0(x), LN1(lat)), q [NB, Q, C] = LN1(lat))."""
    lib = load()
    NB, T, C = x.shape
    Q = lat.shape[1]
    assert tuple(lat.shape) == (NB, Q, C)
    kv = torch.empty((NB, T + Q, C), dtype=torch.float16, device=x.device)
    q = torch.empty_like(lat)
    check(lib.cfgpp_op_ip_ln_concat(ptr(x), ptr(lat), c_int(NB), c_int(T), c_int(Q), c_int(C), ptr(g0), ptr(b0),
                                    ptr(g1), ptr(b1), c_float(eps), ptr(kv), ptr(q), stream_ptr()))
    return kv, q


def op_cfgpp_step(eps_uc: torch.Tensor, eps_c: torch.Tensor, method: int, coef, z: torch.Tensor,
                  aux: torch.Tensor | None = None, want_z0t: bool = True, noise: torch.Tensor | None = None,
                  lambdas: torch.Tensor | None = None):
    """In-place CFG++ update of z (fp32 or fp16 state) from given eps; returns z0t (or None). `noise`: fp16 table
    [slots, *z.shape] of the ancestral samplers (slot = coef.c3). `lambdas`: a per-image guidance table, fp32
    [z.shape[0]] on the device, row b of z mixing with lambdas[b]; None uses coef.lambda_."""
    from ctypes import byref
    lib = load()
    z0t = torch.empty_like(z) if want_z0t else None
    code = 0 if z.dtype == torch.float16 else 1
    if lambdas is not None:
        assert lambdas.dtype == torch.float32 and lambdas.shape == (z.shape[0],)
    check(lib.cfgpp_op_cfgpp_step(ptr(eps_uc), ptr(eps_c), c_int(z.numel()), c_int(method), c_int(code), byref(coef),
                                  ptr(z), ptr(aux), ptr(z0t), ptr(noise), ptr(lambdas), c_int(z.shape[0]),
                                  stream_ptr()))
    return z0t


def op_timestep_embedding(vals: torch.Tensor, n: int, dim: int, out: torch.Tensor | None = None, val_stride: int = 1,
                          col_off: int = 0) -> torch.Tensor:
    """Sinusoidal embedding of the fp32 values vals[i * val_stride], i < n: row i of out gets cos at columns
    [col_off, col_off + dim/2) and sin at [col_off + dim/2, col_off + dim), fp16; other columns are left as they are.
    Without `out`, returns a fresh [n, dim] tensor."""
    lib = load()
    assert vals.dtype == torch.float32 and vals.dim() == 1 and vals.numel() >= (n - 1) * val_stride + 1
    if out is None:
        out = torch.empty((n, dim), dtype=torch.float16, device=vals.device)
    assert out.dtype == torch.float16 and out.dim() == 2 and out.shape[0] >= n and col_off + dim <= out.shape[1]
    check(lib.cfgpp_op_timestep_embedding(ptr(vals), c_int(val_stride), c_int(n), c_int(dim), ptr(out),
                                          c_int(out.stride(0)), c_int(col_off), stream_ptr()))
    return out


def op_small_linear(x: torch.Tensor, w: torch.Tensor, bias=None, addend=None, rows: int | None = None,
                    out_silu: bool = False, want_out2: bool = False):
    """Tiny-M linear: x [R, K] (or [1, K] broadcast to `rows` rows, the kernel's ld_in = 0), w [N, K] fp16. Returns
    (out [R, N], out2 [R, N] = fp16(SiLU(out)) or None)."""
    lib = load()
    K = x.shape[1]
    N = w.shape[0]
    R = x.shape[0] if rows is None else rows
    ld_in = 0 if rows is not None else K
    assert rows is None or x.shape[0] == 1
    assert w.shape[1] == K and (addend is None or addend.shape == (R, N))
    # NaN-filled, so a row or column the kernel fails to write shows
    out = torch.full((R, N), float("nan"), dtype=torch.float16, device=x.device)
    out2 = torch.full_like(out, float("nan")) if want_out2 else None
    check(lib.cfgpp_op_small_linear(ptr(x), c_int(ld_in), ptr(w), ptr(bias), ptr(addend), c_int(N), ptr(out), c_int(N),
                                    ptr(out2), c_int(R), c_int(N), c_int(K), c_int(1 if out_silu else 0),
                                    stream_ptr()))
    return out, out2


def op_copy_rows(src: torch.Tensor, dst: torch.Tensor, rows: int, col_off: int = 0) -> torch.Tensor:
    """dst[r, col_off:col_off + cols] = src[r % src_rows] for r < rows, in place; src [src_rows, cols] fp16."""
    lib = load()
    src_rows, cols = src.shape
    assert dst.dtype == torch.float16 and dst.shape[0] >= rows and col_off + cols <= dst.shape[1]
    check(lib.cfgpp_op_copy_rows(ptr(src), c_int(src_rows), c_int(cols), ptr(dst), c_int(dst.stride(0)),
                                 c_int(col_off), c_int(rows), stream_ptr()))
    return dst


def op_conv_in(z: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, in_scale: torch.Tensor | None = None,
               reps: int = 1) -> torch.Tensor:
    """conv_in 3x3 pad 1: z [B,4,H,W] fp16 / fp32 NCHW (times the device scalar in_scale, fp32 [1], when given),
    w [Cout, 36] fp16 (PyTorch's [Cout,4,3,3] flattened) -> [reps * B, H, W, Cout] NHWC fp16."""
    lib = load()
    B, Cin, H, W = z.shape
    Cout = w.shape[0]
    assert Cin == 4 and w.shape == (Cout, 36)
    assert in_scale is None or (in_scale.dtype == torch.float32 and in_scale.numel() == 1)
    out = torch.empty((reps * B, H, W, Cout), dtype=torch.float16, device=z.device)
    check(lib.cfgpp_op_conv_in(ptr(z), c_int(dtype_code(z)), ptr(in_scale), ptr(w), ptr(bias), ptr(out), c_int(B),
                               c_int(H), c_int(W), c_int(Cout), c_int(reps), stream_ptr()))
    return out


def op_conv_in_add(z: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, addend: torch.Tensor,
                   in_scale: torch.Tensor | None = None, reps: int = 1) -> torch.Tensor:
    """op_conv_in followed by fp16(out + addend), addend [B,H,W,Cout] NHWC fp16 shared by the `reps` repetitions."""
    lib = load()
    B, Cin, H, W = z.shape
    Cout = w.shape[0]
    assert Cin == 4 and w.shape == (Cout, 36) and addend.shape == (B, H, W, Cout) and addend.dtype == torch.float16
    out = torch.empty((reps * B, H, W, Cout), dtype=torch.float16, device=z.device)
    check(lib.cfgpp_op_conv_in_add(ptr(z), c_int(dtype_code(z)), ptr(in_scale), ptr(w), ptr(bias), ptr(addend),
                                   ptr(out), c_int(B), c_int(H), c_int(W), c_int(Cout), c_int(reps), stream_ptr()))
    return out


def op_conv_out_step(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, method: int = 0, coef=None,
                     z: torch.Tensor | None = None, aux: torch.Tensor | None = None, want_z0t: bool = True,
                     noise: torch.Tensor | None = None, lambdas: torch.Tensor | None = None, v_ab=None,
                     in_scale: torch.Tensor | None = None):
    """conv_out 3x3 (Cin -> 4) on x [2B,H,W,Cin] NHWC fp16, w [4, 9, Cin] (`w.permute(0, 2, 3, 1)`), fused with the
    step `method` on the state z [B,4,H,W] (in place). Returns (eps_uc, eps_c, z0t or None); method 0 (STEP_NONE) only
    writes the eps. noise / lambdas as in op_cfgpp_step. `v_ab` = (a, b) of a v-prediction model: the conv outputs are
    v (returned as they are) and become eps = fp16(fp32(a v) + fp32(b x_in)) before the step, x_in = z * in_scale
    (fp32 [1] device scalar, or None) as conv_in forms the UNet input."""
    from ctypes import byref
    lib = load()
    B2, H, W, Cin = x.shape
    B = B2 // 2
    assert B2 == 2 * B and w.shape == (4, 9, Cin)
    eps_uc = torch.empty((B, 4, H, W), dtype=torch.float16, device=x.device)
    eps_c = torch.empty_like(eps_uc)
    z0t = None
    code = 1
    if method != 0:
        assert z is not None and z.shape == (B, 4, H, W) and coef is not None
        z0t = torch.empty_like(z) if want_z0t else None
        code = dtype_code(z)
    if lambdas is not None:
        assert lambdas.dtype == torch.float32 and lambdas.shape == (B,)
    assert in_scale is None or (in_scale.dtype == torch.float32 and in_scale.numel() == 1)
    ab = (c_float * 2)(*v_ab) if v_ab is not None else None
    check(lib.cfgpp_op_conv_out_step(ptr(x), ptr(w), ptr(bias), c_int(B), c_int(H), c_int(W), c_int(Cin),
                                     c_int(method), c_int(code), byref(coef) if coef is not None else c_void_p(0),
                                     ptr(z), ptr(aux), ptr(z0t), ptr(eps_uc), ptr(eps_c), ptr(noise), ptr(lambdas),
                                     ab, ptr(in_scale), stream_ptr()))
    return eps_uc, eps_c, z0t


def op_v_to_eps(v: torch.Tensor, z: torch.Tensor, a: float, b: float, in_scale: torch.Tensor | None = None):
    """eps = fp16(fp32(a v) + fp32(b x_in)), x_in = z * in_scale formed as conv_in forms the UNet input; v fp16, z fp16 /
    fp32 of v's shape."""
    lib = load()
    assert v.dtype == torch.float16 and z.shape == v.shape
    assert in_scale is None or (in_scale.dtype == torch.float32 and in_scale.numel() == 1)
    eps = torch.empty_like(v)
    check(lib.cfgpp_op_v_to_eps(ptr(v), ptr(z), c_int(dtype_code(z)), ptr(in_scale), c_float(a), c_float(b), ptr(eps),
                                c_int(v.numel()), stream_ptr()))
    return eps


def op_upsample2x(x: torch.Tensor) -> torch.Tensor:
    """nearest 2x: x [B,H,W,C] NHWC fp16 -> [B,2H,2W,C]."""
    lib = load()
    B, H, W, C = x.shape
    out = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float16, device=x.device)
    check(lib.cfgpp_op_upsample2x(ptr(x), ptr(out), c_int(B), c_int(H), c_int(W), c_int(C), stream_ptr()))
    return out


def op_image_to_nhwc(x: torch.Tensor, Cp: int) -> torch.Tensor:
    """The ControlNet conditioning image in: x [B,C,H,W] fp16 / fp32 -> [B,H,W,Cp] NHWC fp16, channels C..Cp-1 +0."""
    lib = load()
    B, C, H, W = x.shape
    out = torch.empty((B, H, W, Cp), dtype=torch.float16, device=x.device)
    check(lib.cfgpp_op_image_to_nhwc(ptr(x), c_int(dtype_code(x)), ptr(out), c_int(B), c_int(C), c_int(H), c_int(W),
                                     c_int(Cp), stream_ptr()))
    return out


def op_silu(x: torch.Tensor) -> torch.Tensor:
    """In place on fp16 x: fp16(x / (1 + expf(-x))), the SiLU of the ControlNet conditioning embedding."""
    lib = load()
    assert x.dtype == torch.float16
    check(lib.cfgpp_op_silu(ptr(x), ctypes.c_size_t(x.numel()), stream_ptr()))
    return x


def op_vae_latent_prep(z: torch.Tensor, scaling: float, w: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """fp16(w @ fp16(z / scaling) + bias) per pixel: z [B,4,H,W] fp16 / fp32, w [4, 4] fp16 -> [B,4,H,W] fp16."""
    lib = load()
    B, C, H, W = z.shape
    assert C == 4 and w.shape == (4, 4)
    out = torch.empty((B, 4, H, W), dtype=torch.float16, device=z.device)
    check(lib.cfgpp_op_vae_latent_prep(ptr(z), c_int(dtype_code(z)), c_float(scaling), ptr(w), ptr(bias), ptr(out),
                                       c_int(B), c_int(H * W), stream_ptr()))
    return out


def op_vae_row_softmax(s: torch.Tensor, scale: float) -> torch.Tensor:
    """In-place softmax(s * scale) over the rows of s [rows, n] fp16."""
    lib = load()
    rows, n = s.shape
    check(lib.cfgpp_op_vae_row_softmax(ptr(s), c_int(rows), c_int(n), c_float(scale), stream_ptr()))
    return s


def op_vae_conv_rgb(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """conv 3x3 pad 1, C -> 3: x [B,H,W,C] NHWC fp16, w [3, 9, C] -> [B,3,H,W] NCHW fp16."""
    lib = load()
    B, H, W, C = x.shape
    assert w.shape == (3, 9, C)
    out = torch.empty((B, 3, H, W), dtype=torch.float16, device=x.device)
    check(lib.cfgpp_op_vae_conv_rgb(ptr(x), ptr(w), ptr(bias), ptr(out), c_int(B), c_int(H), c_int(W), c_int(C),
                                    stream_ptr()))
    return out


def op_vae_image_pad(x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """image [B,3,H,W] fp16 / fp32 -> [B,4,H,W] fp16 with a zero fourth plane (into `out` when given)."""
    lib = load()
    B, C, H, W = x.shape
    assert C == 3
    if out is None:
        out = torch.empty((B, 4, H, W), dtype=torch.float16, device=x.device)
    assert out.shape == (B, 4, H, W) and out.dtype == torch.float16 and out.is_contiguous()
    check(lib.cfgpp_op_vae_image_pad(ptr(x), c_int(dtype_code(x)), ptr(out), c_int(B), c_int(H), c_int(W),
                                     stream_ptr()))
    return out


def op_vae_moments_sample(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, wq: torch.Tensor, bq: torch.Tensor,
                          scaling: float, noise: torch.Tensor | None = None) -> torch.Tensor:
    """Encoder tail: conv 3x3 C -> 8 on x [B,H,W,C] NHWC (w [8, 9, C]), quant_conv (wq [8, 8], bq [8]), then
    (mean + exp(clamp(logvar, -30, 20) / 2) * noise) * scaling -> [B,4,H,W] fp32; noise [B,4,H,W] fp16 or None."""
    lib = load()
    B, H, W, C = x.shape
    assert w.shape == (8, 9, C) and wq.shape == (8, 8)
    out = torch.empty((B, 4, H, W), dtype=torch.float32, device=x.device)
    check(lib.cfgpp_op_vae_moments_sample(ptr(x), ptr(w), ptr(bias), ptr(wq), ptr(bq), ptr(noise), c_float(scaling),
                                          ptr(out), c_int(B), c_int(H), c_int(W), c_int(C), stream_ptr()))
    return out


def op_clip_embed(ids: torch.Tensor, tok: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """ids [M] int32 -> [M, D] fp16 = fp16(tok[ids[r]] + pos[r % T]); tok [vocab, D], pos [T, D]."""
    lib = load()
    vocab, D = tok.shape
    T = pos.shape[0]
    assert ids.dtype == torch.int32 and ids.dim() == 1 and pos.shape[1] == D
    out = torch.empty((ids.numel(), D), dtype=torch.float16, device=tok.device)
    check(lib.cfgpp_op_clip_embed(ptr(ids), ptr(tok), ptr(pos), ptr(out), c_int(ids.numel()), c_int(T), c_int(D),
                                  c_int(vocab), stream_ptr()))
    return out


def op_clip_attention(qkv: torch.Tensor, B: int, T: int, heads: int) -> torch.Tensor:
    """Causal self-attention of the CLIP towers: qkv [B*T, 3D] fp16 (q | k | v, 64-wide heads) -> [B*T, D]."""
    lib = load()
    D = qkv.shape[1] // 3
    assert qkv.shape == (B * T, 3 * D)
    out = torch.empty((B * T, D), dtype=torch.float16, device=qkv.device)
    check(lib.cfgpp_op_clip_attention(ptr(qkv), ptr(out), c_int(B), c_int(T), c_int(heads), c_int(D), stream_ptr()))
    return out


def op_clip_activation(x: torch.Tensor, mode: int) -> torch.Tensor:
    """In place on fp16 x (numel % 8 == 0): mode 0 quick_gelu, 1 gelu (erf)."""
    lib = load()
    assert x.dtype == torch.float16
    check(lib.cfgpp_op_clip_activation(ptr(x), ctypes.c_size_t(x.numel()), c_int(mode), stream_ptr()))
    return x


def op_clip_gather_rows(x: torch.Tensor, index: torch.Tensor, T: int) -> torch.Tensor:
    """out[b] = x[b * T + index[b]]: x [B*T, D] fp16, index [B] int32 -> [B, D]."""
    lib = load()
    BT, D = x.shape
    B = index.numel()
    assert index.dtype == torch.int32 and BT == B * T
    out = torch.empty((B, D), dtype=torch.float16, device=x.device)
    check(lib.cfgpp_op_clip_gather_rows(ptr(x), ptr(index), ptr(out), c_int(B), c_int(T), c_int(D), stream_ptr()))
    return out


def op_clip_patchify(image: torch.Tensor, patch: int, Kp: int) -> torch.Tensor:
    """CLIP vision patch rows: image [B,3,S,S] fp16 / fp32 -> [B*(S/patch)^2, Kp] fp16, column (c*P + ky)*P + kx,
    columns 3*P*P..Kp-1 +0."""
    lib = load()
    B, C, S, S2 = image.shape
    assert C == 3 and S == S2 and S % patch == 0
    out = torch.empty((B * (S // patch) ** 2, Kp), dtype=torch.float16, device=image.device)
    check(lib.cfgpp_op_clip_patchify(ptr(image), c_int(dtype_code(image)), ptr(out), c_int(B), c_int(S), c_int(patch),
                                     c_int(Kp), stream_ptr()))
    return out


def op_clip_vision_embed(pe: torch.Tensor, cls: torch.Tensor, pos: torch.Tensor, B: int) -> torch.Tensor:
    """CLIP vision embeddings: pe [B*np, D], cls [D], pos [np + 1, D] fp16 -> [B*(np + 1), D] fp16, row (b, 0) =
    fp16(cls + pos[0]), row (b, 1 + p) = fp16(pe[b*np + p] + pos[1 + p])."""
    lib = load()
    T, D = pos.shape
    assert pe.shape == (B * (T - 1), D) and cls.shape == (D,)
    out = torch.empty((B * T, D), dtype=torch.float16, device=pe.device)
    check(lib.cfgpp_op_clip_vision_embed(ptr(pe), ptr(cls), ptr(pos), ptr(out), c_int(B), c_int(T - 1), c_int(D),
                                         stream_ptr()))
    return out
