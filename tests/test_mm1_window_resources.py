"""mm1_kernel's shared memory is its 48-entry queue window (one row of 64 doubles per entry), the scratch row that takes the
stores of lanes that do not put, and the ziggurat table: 48 x 64 x 8 + 512 + 2 048 = 27 136 B per CTA, in both
instantiations, with no stack.  8 such CTAs + the 1 KB reserved per CTA fill 220 KB of an SM's 228 KB.  Compiles both for
sm_90a and reads ptxas's report (no GPU needed)."""
import re
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import __graft_entry__ as g     # noqa: E402

WINDOW, BLOCK = 48, 64
SMEM = WINDOW * BLOCK * 8 + BLOCK * 8 + 256 * 8

SRC = """#include "queue_model.cuh"
#include "mm1_fast.cuh"
namespace cimba_b200 {
static_assert(MM1_WINDOW == %d && QUEUE_BLOCK == %d, "the window this test sizes");
template __global__ void mm1_kernel<false>(const QueueArgs);
template __global__ void mm1_kernel<true>(const QueueArgs);
}
""" % (WINDOW, BLOCK)


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    d = tmp_path_factory.mktemp("mm1_window")
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
def test_window_shared_memory(ptxas_report, trace):
    text = ptxas_report[trace]
    assert int(re.search(r"(\d+) bytes smem", text).group(1)) == SMEM, text
    assert "0 bytes stack frame" in text, text
