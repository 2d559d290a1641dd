"""NativeUNet — Python owner of one `cfgpp_handle` (one per process and GPU).

Replaces `pipe.unet` of the reference (latent_diffusion.py:67, latent_sdxl.py:50,391) plus the arithmetic between
UNet calls: everything below goes through the C ABI of libcfgpp_b200.so into hand-written sm_90a kernels.
PyTorch only owns the tensors and the stream. There is no eager / CPU fallback.
"""
from __future__ import annotations

import ctypes
from ctypes import POINTER, byref, c_double, c_float, c_int, c_size_t
from typing import Dict, Optional, Sequence

import torch

from . import _native as nv
from .config import UNetConfig, to_desc
from .schedule import F16, F32, StepStateC, to_c_array, v_pred_coefs, v_to_eps


class NativeUNet(nv.NativeHandle):
    _prefix, _what = "", "backend"

    def __init__(self, cfg: UNetConfig, state_dict: Dict[str, torch.Tensor], device="cuda:0"):
        self.cfg = cfg
        # v-prediction (SD 2.x at 768^2): the fused step converts the UNet's v to eps with per-entry (a, b); the un-fused
        # seams (predict_noise here, cfgpp_unet_forward) return the raw model output
        self.v_prediction = cfg.prediction_type == "v_prediction"
        self.v_coefs = None  # (a, b) per entry of the current schedule (v-prediction only)
        self._open(to_desc(cfg), state_dict.items(), device)
        self.batch = 0
        self.latent_hw = (0, 0)
        self._nsteps = 0
        self._state_dtype = torch.float32
        self._bound = None  # strong references to the tensors of the bound prompt (see bind_prompt)
        self._loras = {}  # name -> [adapter id, scale]
        self._lora_per_key = {}  # weight key -> adapters targeting it
        self.controlnet = None  # the attached NativeControlNet (its plan is part of ours)
        self._control_image = None  # the control image embedded for the prepared shape
        self.ip_adapter = None  # the attached ip_adapter.IPAdapter
        self.ip_request = None  # the IPRequest of the running sample() call (bind_control applies it), else None
        self._ip_embeds = None  # the image embeds projected for the prepared plan
        self.t2i_request = None  # the t2i_adapter.T2IRequest of the running sample() call (bind_control applies it)
        self._t2i_n = 0  # T2I-Adapter features the native plan places
        self._t2i_features = None  # the feature list copied into the prepared plan
        self._t2i_flags = None  # the T2I word of every entry of the current schedule, else None

    def _create(self, desc, idx: int) -> None:
        nv.check(self.lib.cfgpp_create_ex(byref(desc), c_size_t(ctypes.sizeof(desc)), c_int(idx), byref(self._h)))

    # ---- plan ------------------------------------------------------------------------------------------------
    def prepare(self, batch: int, h_lat: int, w_lat: int):
        if (batch, (h_lat, w_lat)) == (self.batch, self.latent_hw):
            return
        # a failing native prepare() leaves the handle unprepared: forget the old shape and the bound prompt first so
        # that the next call re-plans instead of running on freed buffers
        self.batch, self.latent_hw, self._nsteps, self._bound = 0, (0, 0), 0, None
        self._control_image = self._ip_embeds = self._t2i_features = None
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_prepare(self._h, c_int(batch), c_int(h_lat), c_int(w_lat)))
        self.batch, self.latent_hw = batch, (h_lat, w_lat)

    @property
    def workspace_bytes(self) -> int:
        n = c_size_t()
        nv.check(self.lib.cfgpp_workspace_bytes(self._h, byref(n)))
        return n.value

    @property
    def forward_flops(self) -> float:
        f = c_double()
        nv.check(self.lib.cfgpp_forward_flops(self._h, byref(f)))
        return f.value

    @property
    def launches_per_step(self) -> int:
        n = c_int()
        nv.check(self.lib.cfgpp_launches_per_step(self._h, byref(n)))
        return n.value

    @property
    def plan_stats(self) -> dict:
        """{'step_flops': executed per fused step, 'prompt_flops' / 'prompt_launches': once per set_prompt}."""
        sf, pf, pl = c_double(), c_double(), c_int()
        nv.check(self.lib.cfgpp_plan_stats(self._h, byref(sf), byref(pf), byref(pl)))
        return {"step_flops": sf.value, "prompt_flops": pf.value, "prompt_launches": pl.value}

    # ---- conditioning ----------------------------------------------------------------------------------------
    def set_prompt(self, ctx: torch.Tensor, pooled: Optional[torch.Tensor] = None,
                   time_ids: Optional[torch.Tensor] = None):
        """ctx = cat([uc, c]) (2*batch, n_ctx, D); pooled (rows, pooled_dim), time_ids (rows, cfg.num_time_ids), rows
        in {batch, 2*batch} (latent_sdxl.py:249-257)."""
        nb = 2 * self.batch
        assert ctx.shape[0] == nb, f"ctx must have 2*batch={nb} rows"
        ctx = ctx.to(self.device, torch.float16).contiguous()
        add_rows = 0
        if pooled is not None:
            pooled = pooled.to(self.device, torch.float16).contiguous()
            time_ids = time_ids.to(self.device, torch.float32).contiguous()
            add_rows = pooled.shape[0]
            assert time_ids.shape == (add_rows, self.cfg.num_time_ids)
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_prompt(self._h, nv.ptr(ctx), c_int(ctx.shape[1]), nv.ptr(pooled),
                                               ctypes.cast(nv.ptr(time_ids), POINTER(c_float)), c_int(add_rows),
                                               nv.stream_ptr()))

        self._bound = None  # a raw set_prompt() invalidates whatever bind_prompt() cached

    def bind_prompt(self, uc: torch.Tensor, c: torch.Tensor, pooled: Optional[torch.Tensor] = None,
                    time_ids: Optional[torch.Tensor] = None, force: bool = False):
        """set_prompt(cat([uc, c]), pooled, time_ids) unless exactly these tensor OBJECTS (identity + in-place version
        counter) are already bound. The engine keeps strong references to them, so an address can never be recycled
        for another prompt while it is the cache key; every solver sharing this engine sees the same truth. Trajectory
        entry points pass force=True (one K/V projection per trajectory, like the reference's per-call text path);
        the identity test only serves the per-step `predict_noise` seam of the k-diffusion / callback loops."""
        cur = (uc, c, pooled, time_ids)
        if not force and self._bound is not None:
            ts, vers = self._bound
            if all(a is b for a, b in zip(ts, cur)) and vers == tuple(None if t is None else t._version for t in cur):
                return
        self.set_prompt(torch.cat([uc, c], dim=0), pooled, None if time_ids is None else time_ids.float())
        self._bound = (cur, tuple(None if t is None else t._version for t in cur))

    # ---- un-fused seam: predict_noise ------------------------------------------------------------------------
    def predict_noise(self, z: torch.Tensor, t: float, in_scale: float = 1.0):
        """The raw model output of both CFG halves (v for a v-prediction model; the solvers convert)."""
        z = z.to(self.device).contiguous()
        eps_uc = torch.empty(z.shape, dtype=torch.float16, device=self.device)
        eps_c = torch.empty_like(eps_uc)
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_unet_forward(self._h, nv.ptr(z), c_int(nv.dtype_code(z)), c_float(float(t)),
                                                 c_float(float(in_scale)), nv.ptr(eps_uc), nv.ptr(eps_c),
                                                 nv.stream_ptr()))
        return eps_uc, eps_c

    def profile_forward(self, z: torch.Tensor, t: float, in_scale: float = 1.0):
        """[(name, kind, flops, ms)] per plan entry of one eager forward (CUDA events around every launch group)."""
        z = z.to(self.device).contiguous()
        max_n, stride = 4096, 96
        n = c_int()
        ms = (c_float * max_n)()
        fl = (c_double * max_n)()
        kd = (c_int * max_n)()
        names = ctypes.create_string_buffer(max_n * stride)
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_profile_forward(self._h, nv.ptr(z), c_int(nv.dtype_code(z)), c_float(float(t)),
                                                    c_float(float(in_scale)), c_int(max_n), byref(n), ms, fl, kd, names,
                                                    c_int(stride), nv.stream_ptr()))
        out = []
        for i in range(n.value):
            nm = names.raw[i * stride:(i + 1) * stride].split(b"\0", 1)[0].decode()
            out.append((nm, kd[i], fl[i], ms[i]))
        return out

    # ---- fused trajectory ------------------------------------------------------------------------------------
    def set_schedule(self, method: int, state_dtype: torch.dtype, steps: Sequence[StepStateC],
                     guidance: Optional[Sequence[float]] = None, control_scales: Optional[Sequence[float]] = None):
        """`guidance`: per-image guidance scales (set_guidance); None leaves the steps' scalar lambda in charge.
        `control_scales`: one ControlNet conditioning scale per entry (set_control_scales); None leaves the scalar."""
        arr = to_c_array(list(steps))
        code = F16 if state_dtype == torch.float16 else F32
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_schedule(self._h, c_int(method), c_int(code), arr, c_int(len(steps)),
                                                 nv.stream_ptr()))
            if self.v_prediction:
                ab = v_pred_coefs(method, list(steps))
                nv.check(self.lib.cfgpp_set_v_coefs(self._h, ab.ctypes.data_as(POINTER(c_float)), c_int(len(steps)),
                                                    nv.stream_ptr()))
                self.v_coefs = ab
        self._nsteps = len(steps)
        self._state_dtype = state_dtype
        self.set_guidance(guidance)
        if control_scales is not None:
            self.set_control_scales(control_scales)
        self._t2i_flags = None
        if self.t2i_request is not None:  # the adapter_conditioning_factor cut, per entry
            self.set_t2i_steps(self.t2i_request.entry_flags(steps))

    def set_guidance(self, guidance: Optional[Sequence[float]] = None):
        """One guidance scale per image of the prepared batch, rounded to fp32, used by every following step (fused
        and `apply_step`) instead of the schedule's scalar; None clears the table."""
        n = 0 if guidance is None else len(guidance)
        if guidance is not None and n != self.batch:
            raise ValueError(f"{n} guidance scales for a prepared batch of {self.batch}")
        arr = (c_float * n)(*[float(g) for g in guidance]) if n else None
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_guidance(self._h, arr, c_int(n), nv.stream_ptr()))

    def set_state(self, z: torch.Tensor):
        z = z.to(self.device, self._state_dtype).contiguous()
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_state(self._h, nv.ptr(z), c_int(nv.dtype_code(z)), nv.stream_ptr()))

    def set_noise(self, noise: torch.Tensor):
        """Ancestral samplers: fp16 noise table (slots, batch, 4, h, w), one slot per step that adds fresh noise."""
        noise = noise.to(self.device, torch.float16).contiguous()
        assert noise.dim() == 5 and tuple(noise.shape[1:]) == (self.batch, 4, *self.latent_hw), "noise table shape"
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_noise(self._h, nv.ptr(noise), c_int(noise.shape[0]), nv.stream_ptr()))

    def run_steps(self, first: int = 0, n: Optional[int] = None):
        n = self._nsteps - first if n is None else n
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_run_steps(self._h, c_int(first), c_int(n), nv.stream_ptr()))

    def get_state(self, which: int = 0) -> torch.Tensor:
        h, w = self.latent_hw
        out = torch.empty((self.batch, 4, h, w), dtype=self._state_dtype, device=self.device)
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_get_state(self._h, c_int(which), nv.ptr(out), nv.stream_ptr()))
        return out

    def apply_step(self, step: int, eps_uc: torch.Tensor, eps_c: torch.Tensor):
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_apply_step(self._h, c_int(step), nv.ptr(eps_uc.contiguous()),
                                               nv.ptr(eps_c.contiguous()), nv.stream_ptr()))

    def run_trajectory(self, method: int, state_dtype: torch.dtype, steps: Sequence[StepStateC], z: torch.Tensor,
                       guidance: Optional[Sequence[float]] = None, noise: Optional[torch.Tensor] = None,
                       control_scales: Optional[Sequence[float]] = None):
        """A whole trajectory from state `z` on the prepared, prompt-bound handle: NFE replays of the step graph with no
        host synchronisation in between. `noise`: the ancestral samplers' table (set_noise); `control_scales`: the
        attached ControlNet's scale per entry. Returns (z0t, zt)."""
        self.set_schedule(method, state_dtype, steps, guidance, control_scales)
        self.set_state(z)
        if noise is not None:
            self.set_noise(noise)
        self.run_steps(0, len(steps))
        return self.get_state(1), self.get_state(0)

    def callback_step(self, i: int, step: StepStateC):
        """Entry i of the current schedule un-fused, so that a callback can see and replace the state: the UNet through
        predict_noise, a v-prediction output turned into eps with the entry's own (a, b) as the fused step does, then
        the step kernel's update. Returns (z0t, zt)."""
        z = self.get_state(0)
        if self._t2i_flags is not None:
            self.set_t2i_active(self._t2i_flags[i])
        eps_uc, eps_c = self.predict_noise(z, step.t, step.in_scale)
        if self.v_prediction:
            a, b = self.v_coefs[i]
            eps_uc, eps_c = v_to_eps(eps_uc, z.half(), a, b), v_to_eps(eps_c, z.half(), a, b)
        self.apply_step(i, eps_uc, eps_c)
        return self.get_state(1), self.get_state(0)

    def close(self):
        if getattr(self, "controlnet", None) is not None:  # the native handle detaches itself; keep both sides in step
            self.controlnet.attached_to = None
            self.controlnet = None
        super().close()

    def bind_control(self, request, zt: torch.Tensor, uc, c, pooled=None, time_ids=None, force: bool = False):
        """Attach (or, with request None, detach) the request's ControlNet, prepare for zt's shape, bind the prompt and
        embed the control image: the engine set-up of one controlled or uncontrolled call. Engines are shared between
        solvers, so an uncontrolled call detaches whatever an earlier call left attached. The IP-Adapter and the
        T2I-Adapter of `ip_request` / `t2i_request` are attached (or detached) the same way."""
        b, _, h, w = zt.shape
        self.attach_controlnet(None if request is None else request.engine)
        ip = self.ip_request
        self.attach_ip_adapter(None if ip is None else ip.adapter)
        t2i = self.t2i_request
        self.attach_t2i(0 if t2i is None else len(t2i.features))
        self.prepare(b, h, w)
        self.bind_prompt(uc, c, pooled, time_ids, force=force)
        if request is not None:
            self.set_control_image(request.image)
        if ip is not None:
            self.set_ip_image_embeds(ip.embeds, force=force)
            self.set_ip_adapter_scale(ip.scale)
        if t2i is not None:
            self.set_t2i_features(t2i.features, force=force)

    # ---- ControlNet ----------------------------------------------------------------------------------------------
    def attach_controlnet(self, cn) -> None:
        """Attach a NativeControlNet (None detaches). A change drops the plan: the next prepare() builds the plan with
        (or without) the ControlNet, so attaching the one already attached costs nothing."""
        if cn is self.controlnet:
            return
        if cn is not None and cn.attached_to is not None:
            cn.attached_to.attach_controlnet(None)
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_attach_controlnet(self._h, cn._h if cn is not None else None))
        if self.controlnet is not None:
            self.controlnet.attached_to = None
        self.controlnet = cn
        if cn is not None:
            cn.attached_to = self
        self.batch, self.latent_hw, self._nsteps, self._bound, self._control_image = 0, (0, 0), 0, None, None

    def set_control_image(self, image: torch.Tensor, force: bool = False) -> None:
        """(batch, 3, 8h, 8w) RGB in [0, 1] for the prepared shape; its conditioning embedding runs once, here. The
        same tensor object (same in-place version) is not embedded again unless `force`."""
        h, w = self.latent_hw
        assert tuple(image.shape) == (self.batch, 3, 8 * h, 8 * w), "control image shape"
        key = (image, image._version)
        if not force and self._control_image is not None and self._control_image[0] is image \
                and self._control_image[1] == key[1]:
            return
        img = image.to(self.device).contiguous()
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_control_image(self._h, nv.ptr(img), c_int(nv.dtype_code(img)),
                                                      nv.stream_ptr()))
        self._control_image = key

    def set_control_scale(self, scale: float) -> None:
        """The conditioning scale of predict_noise and of every step; clears a per-entry table."""
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_control_scale(self._h, c_float(float(scale)), nv.stream_ptr()))

    def set_control_scales(self, scales: Sequence[float]) -> None:
        """One conditioning scale per entry of the current schedule (controlnet.control_scales), read on the device:
        changing it never recaptures the step graph. set_schedule clears it."""
        arr = (c_float * len(scales))(*[float(s) for s in scales])
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_control_scales(self._h, arr, c_int(len(scales)), nv.stream_ptr()))

    # ---- IP-Adapter -------------------------------------------------------------------------------------------
    def attach_ip_adapter(self, adapter) -> None:
        """Load an `ip_adapter.IPAdapter` into this live handle and attach it (None detaches; the UNet's own weights are
        untouched either way). A change drops the plan: the next prepare() builds every attn2 with (or without) the
        image segment, and set_ip_image_embeds must run after it."""
        if adapter is self.ip_adapter:
            return
        with torch.cuda.device(self.device):
            if adapter is None:
                nv.check(self.lib.cfgpp_ip_adapter_clear(self._h))
            else:
                st = nv.stream_ptr()
                for key, w in adapter.weights.items():
                    w = w.detach().to(self.device).contiguous()
                    shape = (ctypes.c_int64 * w.dim())(*w.shape)
                    nv.check(self.lib.cfgpp_ip_adapter_load_weight(self._h, key.encode(), nv.ptr(w), shape,
                                                                   c_int(w.dim()), c_int(nv.dtype_code(w)), st))
                torch.cuda.synchronize(self.device)
                if adapter.resampler is not None:  # IP-Adapter Plus
                    r = adapter.resampler
                    desc = (c_int * 7)(r["num_queries"], r["embed_dim"], r["seq_len"], r["dim"], r["heads"],
                                       r["depth"], r["ff_mult"])  # cfgpp_ip_resampler_desc
                    nv.check(self.lib.cfgpp_ip_adapter_attach_resampler(self._h, desc))
                else:
                    nv.check(self.lib.cfgpp_ip_adapter_attach(self._h, c_int(adapter.n_tokens),
                                                              c_int(adapter.embed_dim)))
        self.ip_adapter = adapter
        self._ip_embeds = None
        self.batch, self.latent_hw, self._nsteps, self._bound, self._control_image = 0, (0, 0), 0, None, None

    def set_ip_image_embeds(self, embeds: torch.Tensor, force: bool = True) -> None:
        """embeds [batch, E]: one image embedding per image of the prepared batch; for an IP-Adapter Plus, the image
        encoder's hidden states [batch, T, E] (IPAdapter.image_embeds gives either). The unconditional half gets what
        diffusers gives it (IPAdapter.image_rows: zeros, or the hidden states of a zero image); the image projection and
        every block's K / V projection run here. With force False, the same tensor object (same in-place version)
        already projected for this plan is not projected again; any other tensor is (a new reference image with the
        same prompt)."""
        plus = self.ip_adapter is not None and self.ip_adapter.resampler is not None
        assert embeds.dim() == (3 if plus else 2) and embeds.shape[0] == self.batch, \
            "one image embedding (Plus: hidden states) per image of the batch"
        key = (embeds, embeds._version)
        if not force and self._ip_embeds is not None and self._ip_embeds[0] is embeds \
                and self._ip_embeds[1] == key[1]:
            return
        if plus:
            rows = self.ip_adapter.image_rows(embeds).to(self.device)
        else:
            e = embeds.to(self.device, torch.float16)
            rows = torch.cat([torch.zeros_like(e), e]).contiguous()
        with torch.cuda.device(self.device):
            fn = self.lib.cfgpp_set_ip_image_hidden_states if plus else self.lib.cfgpp_set_ip_image_embeds
            nv.check(fn(self._h, nv.ptr(rows), nv.stream_ptr()))
        self._ip_embeds = key

    def set_ip_adapter_scale(self, scale: float) -> None:
        """The scale s of every decoupled cross-attention: a device word, so the step graph is never recaptured."""
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_ip_adapter_scale(self._h, c_float(float(scale)), nv.stream_ptr()))

    # ---- T2I-Adapter ------------------------------------------------------------------------------------------
    def attach_t2i(self, n_features: int) -> None:
        """Expect n_features T2I-Adapter features (0 detaches). A change drops the plan: the next prepare() places one
        gated add per feature in the down path, and set_t2i_features must run after it."""
        if n_features == self._t2i_n:
            return
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_t2i_attach(self._h, c_int(n_features)))
        self._t2i_n, self._t2i_features = n_features, None
        self.batch, self.latent_hw, self._nsteps, self._bound, self._control_image = 0, (0, 0), 0, None, None

    def set_t2i_features(self, features: Sequence[torch.Tensor], force: bool = True) -> None:
        """The adapter's features for the prepared batch (t2i_adapter.NativeT2IAdapter.features: (batch, h, w, C) NHWC
        fp16 each), copied into the plan; both CFG halves add the same rows. With force False, the same list object
        already copied for this plan is not copied again."""
        if not force and self._t2i_features is features:
            return
        fs = [f.to(self.device, torch.float16).contiguous() for f in features]
        assert len(fs) == self._t2i_n and all(f.shape[0] == self.batch for f in fs), "one feature row per image"
        ptrs = (ctypes.c_void_p * len(fs))(*[f.data_ptr() for f in fs])
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_t2i_features(self._h, ptrs, nv.stream_ptr()))
        self._t2i_features = features

    def set_t2i_active(self, on: bool) -> None:
        """Whether predict_noise (and every entry of a new schedule) adds the features; clears a per-entry table."""
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_t2i_active(self._h, c_int(1 if on else 0), nv.stream_ptr()))

    def set_t2i_steps(self, flags: Sequence[bool]) -> None:
        """Whether each entry of the current schedule adds the features (t2i_adapter.entry_flags), read on the device:
        changing it never recaptures the step graph. set_schedule clears it; callback_step follows it."""
        arr = (c_int * len(flags))(*[1 if f else 0 for f in flags])
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_set_t2i_steps(self._h, arr, c_int(len(flags)), nv.stream_ptr()))
        self._t2i_flags = list(flags)

    # ---- LoRA adapters ----------------------------------------------------------------------------------------
    MAX_LORAS_PER_WEIGHT = 4

    def add_lora(self, adapter, scale: float = 1.0, name: Optional[str] = None) -> str:
        """Upload the factors of a `lora.LoraAdapter` and merge it at `scale` next to the adapters already loaded.
        Returns its name (`name`, or lora<id>). The bound prompt is dropped: its K/V came from the old weights."""
        idx = len(self._loras)
        name = name or f"lora{idx}"
        if name in self._loras:
            raise ValueError(f"a LoRA named '{name}' is already loaded")
        for key in adapter.targets:
            if self._lora_per_key.get(key, 0) >= self.MAX_LORAS_PER_WEIGHT:
                raise ValueError(f"{key} already carries {self.MAX_LORAS_PER_WEIGHT} LoRA adapters")
        with torch.cuda.device(self.device):
            for key, (down, up, alpha) in adapter.targets.items():
                down = down.to(self.device, torch.float16).contiguous()
                up = up.to(self.device, torch.float16).contiguous()
                nv.check(self.lib.cfgpp_lora_add(self._h, c_int(idx), key.encode(), nv.ptr(down), nv.ptr(up),
                                                 c_int(down.shape[0]), c_float(float(alpha)), c_int(F16),
                                                 nv.stream_ptr()))
                self._lora_per_key[key] = self._lora_per_key.get(key, 0) + 1
        self._loras[name] = [idx, float(scale)]
        self._apply_lora_scales()
        return name

    def set_lora_scales(self, scales: Dict[str, float]) -> None:
        """Re-merge with new scales for the named adapters (the others keep theirs). Always from the pristine weights:
        the result is the one a fresh engine loaded at these scales would hold, bit for bit."""
        for name in scales:
            if name not in self._loras:
                raise KeyError(f"no LoRA named '{name}' (loaded: {sorted(self._loras)})")
        for name, s in scales.items():
            self._loras[name][1] = float(s)
        self._apply_lora_scales()

    def _apply_lora_scales(self) -> None:
        by_id = sorted(self._loras.values())
        arr = (c_float * len(by_id))(*[s for _, s in by_id])
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_lora_set_scales(self._h, arr, c_int(len(by_id)), nv.stream_ptr()))
        self._bound = None

    def clear_lora(self) -> None:
        """Restore the base weights bit for bit and free factors and backups."""
        with torch.cuda.device(self.device):
            nv.check(self.lib.cfgpp_lora_clear(self._h, nv.stream_ptr()))
        self._loras, self._lora_per_key, self._bound = {}, {}, None

    @property
    def loras(self) -> Dict[str, float]:
        """name -> scale of the loaded adapters."""
        return {name: s for name, (_, s) in self._loras.items()}

    @property
    def lora_stats(self) -> dict:
        """{'adapters', 'targets', 'backup_bytes': device memory of the pristine copies, 'bytes_moved': bytes the last
        merge / clear read and wrote (merge and every refreshed packed layout), from shapes}."""
        na, nt, bb, bm = c_int(), c_int(), c_size_t(), c_size_t()
        nv.check(self.lib.cfgpp_lora_stats(self._h, byref(na), byref(nt), byref(bb), byref(bm)))
        return {"adapters": na.value, "targets": nt.value, "backup_bytes": bb.value, "bytes_moved": bm.value}
