"""Build libcfgpp_b200.so (hand-written sm_90a CUDA behind a C ABI) in-tree with nvcc.

    python -m cfgpp_b200.build [--force]

The .so is a build product (git-ignored). There is no JIT and no CPU fallback: if the library is missing the
product path raises.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
OBJ = ROOT / "lib" / "obj"
LIB = ROOT / "lib" / "libcfgpp_b200.so"
INCLUDE = ROOT.parent / "include"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
          "--expt-relaxed-constexpr", "-I", str(INCLUDE), "-I", str(CSRC)]


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _deps_mtime() -> float:
    hdrs = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list(INCLUDE.glob("*.h"))
    return max((h.stat().st_mtime for h in hdrs), default=0.0)


def _compile(src: Path, force: bool, hdr_mtime: float, verbose: bool) -> Path:
    obj = OBJ / (src.stem + ".o")
    if (not force and obj.exists() and obj.stat().st_mtime > src.stat().st_mtime
            and obj.stat().st_mtime > hdr_mtime):
        return obj
    cmd = [NVCC, *ARCH, *CFLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJ.mkdir(parents=True, exist_ok=True)
    # objects built with another compiler, architecture or flags are never reused (mtimes alone cannot tell)
    stamp = OBJ / "flags.txt"
    flags = " ".join([NVCC, *ARCH, *CFLAGS])
    if not stamp.exists() or stamp.read_text() != flags:
        force = True
        stamp.unlink(missing_ok=True)
    srcs = _sources()
    hdr_mtime = _deps_mtime()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, force, hdr_mtime, verbose), srcs))
    newest = max(o.stat().st_mtime for o in objs)
    if force or not LIB.exists() or LIB.stat().st_mtime < newest:
        cmd = [NVCC, *ARCH, "-shared", "-o", str(LIB), *map(str, objs)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(flags)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
