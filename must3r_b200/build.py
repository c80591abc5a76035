"""Build libm3r_b200.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc.

nvcc cross-compiles for sm_90a (H100) without a GPU; the resulting .so and objects are git-ignored build products.
Usage: ``python -m must3r_b200.build [--force]``.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libm3r_b200.so")
SOURCES = ["runtime.cu", "elementwise.cu", "gemm.cu", "gemm_e4m3.cu", "attention.cu", "model.cu", "image.cu", "pointgrid.cu", "slam.cu", "scene.cu", "jpeg.cu", "png.cu"]  # missing files are skipped
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    flags = list(NVCC_FLAGS)
    variant = "trace" if os.environ.get("M3R_TRACE") == "1" else "release"
    if variant == "trace":                               # debug build: in-kernel %globaltimer stamps (tools/trace_*.py)
        flags.append("-DM3R_TRACE")
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "must3r_b200.h"))
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    marker = os.path.join(objdir, ".variant")
    if not os.path.exists(marker) or open(marker).read().strip() != variant:
        force = True                                     # objects of the other variant must not be linked in
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        if force or _stale(obj, [os.path.join(CSRC, src)] + headers):
            cmd = [nvcc] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
            if verbose:
                print(r.stderr)
            return obj, True
        return obj, False

    with ThreadPoolExecutor(max_workers=len(srcs)) as ex:
        res = list(ex.map(compile_one, srcs))
    objs = [o for o, _ in res]
    if force or any(c for _, c in res) or _stale(OUT, objs):
        cmd = [nvcc, "-shared"] + GENCODE + ["-o", OUT] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(marker, "w") as f:
        f.write(variant)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
