"""In-situ timeline of the GEMM kernel at the UNets' transformer shapes: per-CTA globaltimer stamps (prologue, PDL wait,
the MMA warps' end of main loop / start of the next one, the service warps' stores), run back-to-back so A / W are
L2-warm as in the step, plus the CUDA-event time per launch of each shape (and of the GEGLU launch, which the timeline
entry point does not take).

    python tools/gemm_timeline.py [n_shapes]

`mma_gap` is the MMA warps' time between the first tile's last k-block and the second tile's main-loop start: the part
of the epilogue the tensor pipe waits for. Run with CFGPP_B200_LIB pointing at another build to compare two builds
(stamps a build does not write print as absent)."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from cfgpp_b200 import _native as nv  # noqa: E402

dev = torch.device("cuda:0")
lib = nv.load()
# slot -> stamp (slots 1, 3, 4 are not written)
names = {0: "entry", 2: "pdl_wait_done", 5: "tile0_lastkb", 6: "tile1_start", 7: "epiL_lastkb", 8: "epi0_store",
         9: "epiL_start", 10: "epiL_store", 11: "exit", 13: "epiL_staged", 14: "svcL_staged_seen", 15: "svcL_freed"}
SHAPES = [  # (M, N, K, residual, geglu): SDXL batch-4 transformer GEMMs at the 1280- and 640-channel levels
    (4096, 3840, 1280, False, False), (4096, 1280, 1280, True, False), (4096, 10240, 1280, False, True),
    (4096, 1280, 5120, True, False), (16384, 1920, 640, False, False), (16384, 640, 640, True, False),
    (16384, 5120, 640, False, True), (16384, 640, 2560, True, False)]


def event_us(fn, iters=50):
    for _ in range(5):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


print(f"# {torch.cuda.get_device_name(0)}  library {nv.lib_path()}")
for (M, N, K, res, geglu) in SHAPES[: int(sys.argv[1]) if len(sys.argv) > 1 else None]:
    g = torch.Generator().manual_seed(0)
    a = torch.randn(M, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(dev)
    bias = torch.randn(N, generator=g).half().to(dev)
    addend = torch.randn(M, N, generator=g).half().to(dev) if res else None
    us = event_us(lambda: nv.op_linear(a, w, bias, addend, geglu=geglu))
    tf = 2.0 * M * N * K / us / 1e6
    print(f"--- GEMM M={M} N={N} K={K} residual={res} geglu={geglu}: {us:.1f} us per launch, {tf:.0f} TFLOP/s")
    if geglu:
        continue
    out = torch.empty(M, N, dtype=torch.float16, device=dev)
    buf = (C.c_ulonglong * (16 * 132))()
    grid = C.c_int()
    nv.check(lib.cfgpp_dbg_linear_timeline(nv.ptr(a), C.c_int(K), nv.ptr(w), C.c_int(M), C.c_int(N), C.c_int(K),
                                           nv.ptr(bias), nv.ptr(addend), nv.ptr(out), C.c_int(0), C.c_int(10), buf,
                                           C.byref(grid), nv.stream_ptr()))
    t = np.array(buf[: 16 * grid.value], dtype=np.uint64).reshape(grid.value, 16).astype(np.int64)
    t0 = t[:, 0].min()
    items = t[:, 12]
    print(f"   grid={grid.value} kernel span {(t[:, 11].max() - t0) / 1e3:.1f} us, tiles/CTA max {items.max()} "
          f"min {items.min()}")
    for i, nm in names.items():
        col = t[:, i]
        valid = col > 0
        if valid.any():
            rel = (col[valid] - t0) / 1e3
            print(f"   {nm:16s} mean {rel.mean():7.2f}  min {rel.min():7.2f}  max {rel.max():7.2f} us  (n={valid.sum()})")
        else:
            print(f"   {nm:16s} absent")
    two = (t[:, 5] > 0) & (t[:, 6] > 0)
    if two.any():
        gap = (t[two, 6] - t[two, 5]) / 1e3
        tile = (t[two, 7] - t[two, 5]) / 1e3 / np.maximum(items[two] - 1, 1)
        print(f"   mma_gap (tile 0 last k-block -> tile 1 start) mean {gap.mean():.2f} min {gap.min():.2f} "
              f"max {gap.max():.2f} us; tile period {tile.mean():.2f} us")
    # the epilogue of the last tile, as both builds stamp it: vectors ready -> store issued
    lst = (t[:, 9] > 0) & (t[:, 10] > 0)
    if lst.any():
        print(f"   last tile epiL_start -> epiL_store mean {((t[lst, 10] - t[lst, 9]) / 1e3).mean():.2f} us")
