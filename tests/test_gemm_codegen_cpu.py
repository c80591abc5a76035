"""Generated-code guard for the warp-specialised wgmma kernels (no GPU needed): compiles gemm.cu and attention.cu with the
library's nvcc flags plus -Xptxas -v and checks what ptxas reports.

- No spill stores or loads and no stack frame in any instantiation: the consumer warpgroups hold a 64 x BN fp32
  accumulator (128 registers at BN = 256) and rely on the setmaxnreg register split to keep it and the epilogue in
  registers.
- No warning C7519 ("warpgroup.arrive is injected ... to allow use of registers in GMMA"): ptxas injects it when it
  cannot keep the accumulator registers untouched between wgmma groups, and then serialises the main loop."""
import os
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from must3r_b200 import build as b

GEMM_INSTANTIATIONS = 22     # (BN, mode) pairs {32..256 plain, 64 / 128 LayerNorm-emitting, 64 / 128 / 256 grouped} x fp16 / bf16


def _ptxas_report(src, out_dir):
    cmd = [b._nvcc()] + b.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(b.CSRC, src), "-o", os.path.join(out_dir, src + ".o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed for {src}:\n{r.stderr}"
    return r.stdout + r.stderr


def _per_kernel(report):
    """{mangled entry name: (stack frame, spill stores, spill loads)} from ptxas -v output."""
    out, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = tuple(int(v) for v in m.groups())
            cur = None
    return out


@pytest.fixture(scope="module")
def reports(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("codegen"))
    with ThreadPoolExecutor(max_workers=2) as ex:
        gemm, attn = ex.map(lambda s: _ptxas_report(s, d), ["gemm.cu", "attention.cu"])
    return {"gemm": gemm, "attention": attn}


def test_gemm_kernels_do_not_spill(reports):
    kernels = {k: v for k, v in _per_kernel(reports["gemm"]).items() if "gemm_kernel" in k}
    assert len(kernels) == GEMM_INSTANTIATIONS, sorted(kernels)
    bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
    assert not bad, f"(stack frame, spill stores, spill loads) bytes: {bad}"


def test_gemm_main_loop_is_not_serialised(reports):
    hits = re.findall(r"C7519.*", reports["gemm"])
    assert not hits, "\n".join(hits[:5])


def test_attention_kernels_do_not_spill(reports):
    kernels = {k: v for k, v in _per_kernel(reports["attention"]).items() if "attn_kernel" in k}
    assert len(kernels) == 2, sorted(kernels)
    bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
    assert not bad, f"(stack frame, spill stores, spill loads) bytes: {bad}"
    assert "C7519" not in reports["attention"]
