"""In-situ timeline of the GEMM kernel: per-CTA globaltimer stamps (prologue, PDL wait, first data, per-tile main
loop / epilogue, exit) for a few of the UNet's GEMM shapes, run back-to-back so A / W are L2-warm as in the step."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from cfgpp_b200 import _native as nv  # noqa: E402

dev = torch.device("cuda:0")
lib = nv.load()
names = ["entry", "prologue_done", "pdl_wait_done", "first_tma", "first_full", "tile0_lastkb", "lasttile_lastkb",
         "sk_preload_done", "epi0_store", "epiL_start", "epiL_store", "exit", "ntiles", "sk_fin_wait", "sk_fin_seen", "sk_part_published"]
for (M, N, K, res, bn) in [(4096, 1280, 1280, False, 0), (4096, 1280, 1280, True, 0), (4096, 1280, 5120, True, 0),
                           (4096, 3840, 1280, False, 0), (16384, 640, 640, True, 0), (8192, 8192, 8192, False, 256)
                           ][: int(sys.argv[1]) if len(sys.argv) > 1 else None]:
    g = torch.Generator().manual_seed(0)
    a = torch.randn(M, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(dev)
    bias = torch.randn(N, generator=g).half().to(dev) if res else None
    addend = torch.randn(M, N, generator=g).half().to(dev) if res else None
    out = torch.empty(M, N, dtype=torch.float16, device=dev)
    buf = (C.c_ulonglong * (16 * 132))()
    grid = C.c_int()
    nv.check(lib.cfgpp_dbg_linear_timeline(nv.ptr(a), C.c_int(K), nv.ptr(w), C.c_int(M), C.c_int(N), C.c_int(K),
                                           nv.ptr(bias), nv.ptr(addend), nv.ptr(out), C.c_int(bn), C.c_int(10), buf,
                                           C.byref(grid), nv.stream_ptr()))
    t = np.array(buf[: 16 * grid.value], dtype=np.uint64).reshape(grid.value, 16).astype(np.int64)
    t0 = t[:, 0].min()
    print(f"--- GEMM M={M} N={N} K={K} residual={res} grid={grid.value}  kernel span {(t[:, 11].max() - t0)/1e3:.1f} us "
          f"tiles/CTA max {t[:, 12].max()} min {t[:, 12].min()}")
    for i, nm in enumerate(names):
        if nm == 'ntiles':
            continue
        col = t[:, i]
        valid = col > 0
        if valid.any():
            rel = (col[valid] - t0) / 1e3
            print(f"   {nm:16s} mean {rel.mean():7.2f}  min {rel.min():7.2f}  max {rel.max():7.2f} us  (n={valid.sum()})")
    for cta in (0, 1, 2, 3, 40, 41, 146, 147):
        if cta < grid.value:
            print(f"   cta {cta:3d}: " + " ".join(f"{nm}={(t[cta, i] - t0) / 1e3:.1f}" for i, nm in enumerate(names)
                                              if nm != 'ntiles' and t[cta, i] > 0) + f" items={t[cta, 12]}")
