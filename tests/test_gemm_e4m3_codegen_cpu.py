"""Generated-code guard for the e4m3 wgmma GEMM (no GPU needed): gemm_e4m3.cu compiled with the library's flags and
-Xptxas -v.  Every instantiation (plain and grouped, tile widths 64 / 128 / 256) keeps its accumulator and epilogue in
registers (no stack frame, no spills), fits the setmaxnreg split's launch budget, and ptxas does not serialise the k loop
(warning C7519); in the SASS the four k32 wgmma of a k-block issue back to back."""
import os
import re
import subprocess

import pytest

from must3r_b200 import build as b
from test_gemm_codegen_cpu import _per_kernel, _ptxas_report

E4M3_INSTANTIATIONS = 6
LAUNCH_REGS = (65536 // 384) // 8 * 8          # gemm_kernel.cuh GEMM_LAUNCH_REGS


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    return _ptxas_report("gemm_e4m3.cu", str(tmp_path_factory.mktemp("codegen8")))


def test_e4m3_kernels_do_not_spill(report):
    kernels = {k: v for k, v in _per_kernel(report).items() if "gemm_kernel" in k}
    assert len(kernels) == E4M3_INSTANTIATIONS, sorted(kernels)
    assert all("Li2EE" in k for k in kernels), sorted(kernels)          # OP_E4M3 instantiations only
    bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
    assert not bad, f"(stack frame, spill stores, spill loads) bytes: {bad}"
    regs = [int(r) for r in re.findall(r"Used (\d+) registers", report)]
    assert regs and max(regs) <= LAUNCH_REGS


def test_e4m3_main_loop_is_not_serialised(report):
    assert "C7519" not in report


def test_e4m3_wgmma_issue_back_to_back(tmp_path):
    """Between the four QGMMA of a k-block there is no warpgroup arrive or wait: they form one wgmma group, only its
    last instruction sets the scoreboard (gsb0) that the wait of the next k-block reads."""
    obj = str(tmp_path / "g8.o")
    subprocess.check_call([b._nvcc()] + b.NVCC_FLAGS + ["-c", os.path.join(b.CSRC, "gemm_e4m3.cu"), "-o", obj])
    sass = subprocess.check_output([os.path.join(os.path.dirname(b._nvcc()), "cuobjdump"), "-sass", obj], text=True)
    seq = [ln.split(";")[0].split("*/")[-1].strip() for ln in sass.splitlines() if re.search(r"\b(QGMMA|WARPGROUP)\.", ln)]
    q = [x for x in seq if x.startswith("QGMMA")]
    assert q and all(".E4M3.E4M3" in x for x in q), seq[:6]
    runs, cur = [], []
    for x in seq:
        if x.startswith("QGMMA"):
            cur.append(x)
        elif cur:
            runs.append(cur)
            cur = []
    assert runs and all(len(r) == 4 for r in runs), [len(r) for r in runs]
    assert all("gsb0" in r[-1] and not any("gsb0" in x for x in r[:-1]) for r in runs)
