"""What ptxas made of mm1_kernel's event loop (no GPU needed): both instantiations compiled for sm_90a.

The launch fills an H100 in one wave only while 8 CTAs of 64 threads fit an SM, so the kernel may use at most 128 registers,
no stack and no spills, and its shared memory stays at the 27 136 B of the 48-entry window.  In the loop, a divergent branch
costs a BSSY / BSYNC reconvergence region, and ptxas does not schedule instructions across one, so the event steps overlap
only between regions.  The pop, the bodies and the insert of the wake-up are predicated; an event step keeps two regions, the
look-ahead refill and the rare queue-spill branch, and the parked-set block adds its two nested ones."""
import re
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import __graft_entry__ as g     # noqa: E402

MAX_REGS = 65_536 // (8 * 64)   # 8 CTAs of 64 threads per SM
SMEM = 27_136
MM1_STEPS = 8                   # mm1_fast.cuh: event steps per loop iteration
STEP_REGIONS = 2                # the look-ahead refill and the queue-spill branch
PARK_REGIONS = 2                # the parked-set block: the ballot's branch and the slow path inside it

SRC = """#include "queue_model.cuh"
#include "mm1_fast.cuh"
namespace cimba_b200 {
template __global__ void mm1_kernel<false>(const QueueArgs);
template __global__ void mm1_kernel<true>(const QueueArgs);
}
"""


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    d = tmp_path_factory.mktemp("mm1_sass")
    (d / "mm1.cu").write_text(SRC)
    flags = [f for f in g.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    cubin = d / "mm1.cubin"
    cmd = [g._nvcc(), *flags, "-Xptxas", "-v", "-I", str(g.CSRC), "-I", str(ROOT / "include"), "-cubin",
           "-o", str(cubin), str(d / "mm1.cu")]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    report = {}
    for m in re.finditer(r"Compiling entry function '(\w*mm1_kernelILb([01])E\w*)' for 'sm_90a'\n(.*?)(?=ptxas info\s+: Compile time)",
                         p.stderr, re.S):
        report[m.group(2) == "1"] = m.group(3)
    assert set(report) == {False, True}, p.stderr
    cuobjdump = Path(g._nvcc()).with_name("cuobjdump")
    sass = subprocess.run([str(cuobjdump) if cuobjdump.exists() else "cuobjdump", "-sass", str(cubin)],
                          capture_output=True, text=True, check=True).stdout
    return report, sass


def _loop(sass, trace):
    """The instructions of the event loop: those inside the backward branch with the largest span."""
    blocks = re.split(r"\n\s*Function : ", sass)
    body = [b for b in blocks if f"mm1_kernelILb{int(trace)}E" in b.split("\n", 1)[0]]
    assert len(body) == 1
    ins = [(int(m.group(1), 16), m.group(2).strip())
           for m in re.finditer(r"/\*([0-9a-f]{4,6})\*/\s+([^;]*);", body[0])]
    back = [(t, a) for a, text in ins for t in [re.search(r"BRA\s+(?:`\(\.L_x_\d+\)|0x([0-9a-f]+))", text)]
            if t and t.group(1) and int(t.group(1), 16) < a]
    assert back, "no backward branch"
    start, end = max(((int(t.group(1), 16), a) for t, a in back), key=lambda se: se[1] - se[0])
    return [text for a, text in ins if start <= a <= end]


@pytest.mark.parametrize("trace", [False, True])
def test_registers_stack_and_shared_memory(built, trace):
    text = built[0][trace]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, text
    assert int(re.search(r"Used (\d+) registers", text).group(1)) <= MAX_REGS, text
    assert int(re.search(r"(\d+) bytes smem", text).group(1)) == SMEM, text


def test_event_step_branch_regions(built):
    loop = _loop(built[1], False)
    regions = sum(1 for t in loop if re.match(r"(@!?U?P\w+\s+)?BSSY\b", t))
    assert regions <= STEP_REGIONS * MM1_STEPS + PARK_REGIONS, regions
