"""CPU tests of the last fixed-process coverage models on the static tier's second form (cimba_b200/csrc/cmb_static.cuh, models
with static_interrupts): PoolFightT (model 4: mice that change their own priority and acquire from a pool, rats that pre-empt,
a cat that interrupts, partial releases, cmb_resourcepool_held_by_process) and WorkshopT (models 5 and 12: a cmb_buffer with
partial puts and gets under waiters with priorities, a polite and a pre-empting worker on one cmb_resource, a nuisance that
interrupts with priorities -5..5; model 12 is test/test_buffer.c as it stands, with the level history on).

The models are compiled for the host from one template on the general engine and on the static tier
(tests/static_coverage_host.cpp).  The static tier must reproduce, trial for trial, what the unmodified reference produced: the
vectors of tests/golden/cmb_engine_vectors.json with their pop traces, the golden file test/reference/buffer.txt, and the live
reference build where present.  With one spare event slot it must flag a trial for the general engine, never answer differently."""
import ctypes as C
import random
import re
import struct
import subprocess
import sys
from pathlib import Path

import pytest

from cmb_cases import GOLD, MASTER, TRACE, case_id, check_trial, inverse_fmix64

ROOT = Path(__file__).resolve().parents[1]
GENERAL, STATIC, ONE_SLOT = 0, 1, 2         # host_coverage_run_trials' engines
MODELS = (4, 5, 12)
CASES = [c for c in GOLD["cases"] if c["model"] in MODELS]
REPORTS_FEL = (4, 5)                        # model 12 reports its history's sample count instead


class HostResult(C.Structure):
    _fields_ = [("events", C.c_uint64), ("objects", C.c_uint64), ("t_end", C.c_double), ("sum_wait", C.c_double),
                ("max_fel", C.c_uint64), ("max_queue", C.c_uint64), ("counter", C.c_uint64 * 8), ("status", C.c_uint32),
                ("pad", C.c_uint32)]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = tmp_path_factory.mktemp("coverage") / "libstatic_coverage_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                    "-shared", "-fPIC", str(ROOT / "tests/static_coverage_host.cpp"), "-o", str(so)], check=True, capture_output=True)
    f = C.CDLL(str(so)).host_coverage_run_trials
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double,
                  C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double), C.POINTER(HostResult)]
    return f


def run_host(f, model, engine, case, n, master=MASTER, first=0, trace=TRACE):
    out = (HostResult * n)()
    keys = (C.c_uint64 * max(1, n * trace))()
    times = (C.c_double * max(1, n * trace))()
    rc = f(model, engine, case["servers"], master, first, n, case["num_objects"], float.fromhex(case["arr_mean"]),
           float.fromhex(case["srv_mean"]), 1 << 26, trace, keys, times, out)
    assert rc == 0
    return out, keys, times


def row(o):
    return (o.events, o.objects, o.t_end, o.sum_wait, o.max_queue, list(o.counter))


def _double(u):
    return struct.unpack("<d", struct.pack("<Q", int(u) & (2**64 - 1)))[0]


def check_vector(model, out, keys, times, i, want):
    check_trial(want, out[i].events, out[i].objects, out[i].t_end, out[i].sum_wait, list(out[i].counter),
                keys[i * TRACE:(i + 1) * TRACE], times[i * TRACE:(i + 1) * TRACE], f"trial {i}")
    assert [int(v) for v in out[i].counter] == want["counters8"], (i, "all eight counters")
    if model in REPORTS_FEL:
        assert out[i].max_queue == want["max_fel"], (i, "fel_high")


@pytest.mark.parametrize("case", CASES, ids=case_id)
@pytest.mark.parametrize("engine", [GENERAL, STATIC], ids=["general", "static"])
def test_coverage_models_on_the_cpu_match_the_reference_vectors(host, engine, case):
    """Every vector case of models 4, 5 and 12: events, objects, clock, sums, all eight counters, fel_high where the model reports
    it, the 2000-pop trace, status 0."""
    n = len(case["trials"])
    out, keys, times = run_host(host, case["model"], engine, case, n)
    for i, want in enumerate(case["trials"]):
        assert out[i].status == 0, (i, out[i].status)
        check_vector(case["model"], out, keys, times, i, want)


def test_the_vectors_exercise_what_they_claim():
    """The stored trials pre-empt (model 4's rats, model 5's worker), interrupt, and leave puts and gets of the buffer unfinished."""
    total = {m: [sum(t["counters8"][k] for c in CASES if c["model"] == m for t in c["trials"]) for k in range(8)] for m in MODELS}
    assert total[4][1] > 0 and total[4][2] > 0 and total[4][3] > 0, total[4]      # rats' grabs, pre-empted, interrupted
    assert total[5][2] > 0 and total[5][3] > 0 and total[5][5] > 0, total[5]      # puts and gets cut short, pre-empted worker
    assert total[12][2] > 0 and total[12][3] > 0, total[12]


def test_static_tier_reproduces_the_reference_buffer_golden_file(host):
    """test/reference/buffer.txt on the static tier: the reference's seed, capacity 10, 10 000 time units, level history N 41876,
    time-weighted mean 4.980."""
    case = {"servers": 10, "num_objects": 10_000, "arr_mean": (1.0).hex(), "srv_mean": (1.0).hex()}
    out, _, _ = run_host(host, 12, STATIC, case, 1, master=inverse_fmix64(0x34F05C64D7AD598F), trace=0)
    assert out[0].status == 0 and out[0].max_queue == 41876 and "%.3f" % _double(out[0].counter[4]) == "4.980"
    general, _, _ = run_host(host, 12, GENERAL, case, 1, master=inverse_fmix64(0x34F05C64D7AD598F), trace=0)
    assert row(out[0]) == row(general[0])


def test_static_equals_general_equals_the_live_reference_on_drawn_parameters(host):
    """Models 4, 5 and 12 at drawn capacities 1..40, durations and (for 5 and 12) means: the static tier, the general engine and
    the live reference build (oracle/_ref/librefdrv.so) give the same events, objects, clock, sums, counters and max_queue for
    every trial (max_queue is fel_high for models 4 and 5, the level history's sample count for model 12)."""
    from oracle_libs import load_ref, run_trials
    ref = load_ref()
    rnd = random.Random(20261016)
    for model in MODELS:
        for _ in range(4):
            servers, nobj = rnd.randint(1, 40), rnd.randint(20, 600)
            arr, srv = (1.0, 1.0) if model == 4 else (rnd.choice([0.5, 1.0, 1.5]), rnd.choice([0.5, 1.0, 2.0]))
            case = {"servers": servers, "num_objects": nobj, "arr_mean": arr.hex(), "srv_mean": srv.hex()}
            first = rnd.randint(0, 5000)
            general, _, _ = run_host(host, model, GENERAL, case, 6, first=first, trace=0)
            static, _, _ = run_host(host, model, STATIC, case, 6, first=first, trace=0)
            want = run_trials(ref, "ref", model, servers, MASTER, first, 6, nobj, arr, srv, par=0) if ref is not None else None
            for i in range(6):
                assert static[i].status == 0 and general[i].status == 0, (model, case, i)
                assert row(static[i]) == row(general[i]), (model, case, i)
                if want is not None:
                    w = want[i]
                    assert row(static[i]) == (w.events, w.objects, w.t_end, w.sum_wait, w.max_fel if model in REPORTS_FEL else w.max_queue,
                                              list(w.counter)), (model, case, i)
    if ref is None:
        pytest.skip("oracle/_ref/librefdrv.so not built (needs the reference sources): static = general checked only")


def test_one_spare_slot_flags_the_trial_and_never_answers_differently(host):
    """One spare event slot, where the routes give model 4 four and models 5 and 12 two: each vector trial is either flagged for
    the general engine, or its answer is the reference's exactly - and some flag."""
    flagged = exact = 0
    for case in CASES:
        k = len(case["trials"])
        out, keys, times = run_host(host, case["model"], ONE_SLOT, case, k)
        for i, want in enumerate(case["trials"]):
            if out[i].status:
                flagged += 1
                continue
            exact += 1
            check_vector(case["model"], out, keys, times, i, want)
    assert flagged > 0, (flagged, exact)


# ---- registers, stack and spills of the new static-tier instantiations (no GPU needed)
KERNELS = {"PoolFightT": (6, "models::POOLFIGHT_SPARE_SLOTS"), "WorkshopBufferT": (7, "models::WORKSHOP_SPARE_SLOTS"),
           "WorkshopRecordedT": (7, "models::WORKSHOP_SPARE_SLOTS")}
SRC = """#include "cmb_launch.cuh"
#include "../models/coverage_models.cuh"
#include "../models/workshop_model.cuh"
namespace cimba_b200 { namespace cmb {
""" + "".join(f"template __global__ void static_trial_kernel<models::{m}, {p}, 0, {e}, {t}>(const StaticArgs);\n"
              for m, (p, e) in KERNELS.items() for t in ("false", "true")) + "}}\n"


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    sys.path.insert(0, str(ROOT))
    import __graft_entry__ as g
    d = tmp_path_factory.mktemp("coverage_resources")
    (d / "k.cu").write_text(SRC)
    flags = [f for f in g.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    cmd = [g._nvcc(), *flags, "-Xptxas", "-v", "-I", str(g.CSRC), "-I", str(ROOT / "include"), "-cubin", "-o", str(d / "k.cubin"),
           str(d / "k.cu")]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    report = {}
    for m in re.finditer(r"Compiling entry function '\w*static_trial_kernelINS_6models\d+(\w+?)ELi\d+ELi0ELi\d+ELb([01])E\w*' "
                         r"for 'sm_90a'\n(.*?)(?=ptxas info\s+: Compile time)", p.stderr, re.S):
        report[(m.group(1), m.group(2) == "1")] = m.group(3)
    assert set(report) == {(m, t) for m in KERNELS for t in (False, True)}, p.stderr
    return report


@pytest.mark.parametrize("trace", [False, True])
@pytest.mark.parametrize("model", list(KERNELS))
def test_new_instantiations_build_without_spills(ptxas_report, model, trace):
    """The control block may live on the stack (the guard heaps are indexed at run time); nothing may spill."""
    text = ptxas_report[(model, trace)]
    stack = re.search(r"(\d+) bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", text)
    regs = re.search(r"Used (\d+) registers", text)
    assert stack and regs and int(regs.group(1)) <= 255, text
    print(f"{model} trace={trace}: {regs.group(1)} registers, {stack.group(1)} bytes stack")
