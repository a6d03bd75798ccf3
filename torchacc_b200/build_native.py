"""In-tree build of the native library ``torchacc_b200/_C.so``.

Every ``csrc/**/*.cu`` translation unit is compiled with nvcc for sm_90a only
(``-gencode arch=compute_90a,code=sm_90a -lineinfo``) and linked into one shared object that Python loads
with ctypes.  The kernels do not include PyTorch headers, so a full rebuild takes well under a minute and
works on hosts without a GPU (nvcc cross-compiles).  Objects are cached by source mtime under ``build/obj``.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "csrc"
OBJ = ROOT / "build" / "obj"
OUT = ROOT / "torchacc_b200" / "_C.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _sources():
    return sorted(p for p in CSRC.rglob("*.cu") if "tests" not in p.parts)


def _headers_mtime() -> float:
    hs = list(CSRC.rglob("*.h")) + list(CSRC.rglob("*.cuh"))
    return max((h.stat().st_mtime for h in hs), default=0.0)


def build(verbose: bool = False, force: bool = False, jobs: int | None = None) -> Path:
    nvcc = _nvcc()
    OBJ.mkdir(parents=True, exist_ok=True)
    hdr_m = _headers_mtime()
    todo, objs = [], []
    for src in _sources():
        obj = OBJ / (str(src.relative_to(CSRC)).replace("/", "__")[:-3] + ".o")
        objs.append(obj)
        if force or not obj.exists() or obj.stat().st_mtime < max(src.stat().st_mtime, hdr_m):
            todo.append((src, obj))

    def compile_one(item):
        src, obj = item
        cmd = [nvcc, *NVCC_FLAGS, "-I", str(CSRC), "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    if todo:
        with ThreadPoolExecutor(max_workers=jobs or min(8, os.cpu_count() or 4)) as ex:
            list(ex.map(compile_one, todo))
    if todo or not OUT.exists() or force:
        cmd = [nvcc, "-shared", "-o", str(OUT), *map(str, objs), "-lcudart", "-gencode",
               "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return OUT


if __name__ == "__main__":
    out = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(out)
