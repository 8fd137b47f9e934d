"""mm1_kernel's launch fills an H100 in one wave only if all 8 of its 64-thread CTAs fit on an SM: 8 x 64 lanes x 132 SMs
>= 65 536 trials.  Its static shared memory (ziggurat table, object-queue windows, scratch row) plus the 1 KB the hardware
reserves per CTA must fit 8 times into the SM's 228 KB, and its registers must not spill.  This compiles both instantiations
for sm_90a and reads ptxas's report (no GPU needed)."""
import re
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import __graft_entry__ as g     # noqa: E402

SM_SMEM = 233_472               # 228 KB of shared memory per SM (sm_90)
CTA_RESERVED = 1024             # reserved by the hardware per resident CTA
CTAS_PER_SM = 8
REGS_PER_SM = 65_536

SRC = """#include "queue_model.cuh"
#include "mm1_fast.cuh"
namespace cimba_b200 {
template __global__ void mm1_kernel<false>(const QueueArgs);
template __global__ void mm1_kernel<true>(const QueueArgs);
}
"""


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    d = tmp_path_factory.mktemp("mm1_resources")
    (d / "mm1.cu").write_text(SRC)
    flags = [f for f in g.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    cmd = [g._nvcc(), *flags, "-Xptxas", "-v", "-I", str(g.CSRC), "-I", str(ROOT / "include"), "-cubin",
           "-o", str(d / "mm1.cubin"), str(d / "mm1.cu")]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    report = {}
    for m in re.finditer(r"Compiling entry function '(\w*mm1_kernelILb([01])E\w*)' for 'sm_90a'\n(.*?)(?=ptxas info\s+: Compile time)",
                         p.stderr, re.S):
        report[m.group(2) == "1"] = m.group(3)
    assert set(report) == {False, True}, p.stderr
    return report


@pytest.mark.parametrize("trace", [False, True])
def test_no_spills(ptxas_report, trace):
    text = ptxas_report[trace]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, text


@pytest.mark.parametrize("trace", [False, True])
def test_eight_ctas_fit_an_sm(ptxas_report, trace):
    text = ptxas_report[trace]
    smem = int(re.search(r"(\d+) bytes smem", text).group(1))
    regs = int(re.search(r"Used (\d+) registers", text).group(1))
    assert CTAS_PER_SM * (smem + CTA_RESERVED) <= SM_SMEM, (smem, text)
    assert CTAS_PER_SM * 64 * regs <= REGS_PER_SM, (regs, text)
