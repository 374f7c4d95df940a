"""In-tree build of libsurya_b200.so (sm_90a only: the kernels use Hopper's wgmma, TMA and clusters).

`nvcc -gencode arch=compute_90a,code=sm_90a` cross-compiles without a GPU, so the same function builds the
library on a machine without one.  Objects are cached under `surya_b200/csrc/build/` (git-ignored) keyed by
source + header mtimes; the shared library lands in `surya_b200/lib/` (git-ignored).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OBJDIR = CSRC / "build"
LIBDIR = PKG / "lib"
LIBNAME = "libsurya_b200.so"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
    "-I", str(PKG.parent / "include"),
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: surya_b200 needs the CUDA toolkit to build its sm_90a kernels")


def _newest_header_mtime() -> float:
    hdrs = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list((PKG.parent / "include").glob("*.h"))
    return max((h.stat().st_mtime for h in hdrs), default=0.0)


def lib_path() -> Path:
    return LIBDIR / LIBNAME


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu under csrc/ and link lib/libsurya_b200.so. Returns the library path."""
    nvcc = _nvcc()
    OBJDIR.mkdir(parents=True, exist_ok=True)
    LIBDIR.mkdir(parents=True, exist_ok=True)
    srcs = sorted(CSRC.glob("*.cu"))
    if not srcs:
        raise RuntimeError(f"no CUDA sources under {CSRC}")
    hdr_m = _newest_header_mtime()
    # objects built with other flags (another architecture) are stale whatever their mtime
    flags_file = OBJDIR / "nvcc_flags.txt"
    flags = "\n".join(NVCC_FLAGS)
    if not flags_file.exists() or flags_file.read_text() != flags:
        force = True
    jobs = []
    objs = []
    for src in srcs:
        obj = OBJDIR / (src.stem + ".o")
        objs.append(obj)
        stale = force or (not obj.exists()) or obj.stat().st_mtime < max(src.stat().st_mtime, hdr_m)
        if stale:
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = (r.stdout or "") + (r.stderr or "")
        (OBJDIR / (src.stem + ".log")).write_text(log)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{log[-4000:]}")
        return src.name

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for name in ex.map(compile_one, jobs):
                if verbose:
                    print(f"[surya_b200.build] compiled {name}", file=sys.stderr)

    flags_file.write_text(flags)
    lib = lib_path()
    if jobs or not lib.exists() or any(o.stat().st_mtime > lib.stat().st_mtime for o in objs):
        cmd = [nvcc, "-shared", *GENCODE, "-o", str(lib), *map(str, objs)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(f"[surya_b200.build] linked {lib}", file=sys.stderr)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
