"""CPU tests of the static tier's second form (cimba_b200/csrc/cmb_static.cuh, a model with static_interrupts): process
priorities, cmb_process_interrupt, CMB_RESOURCEPOOL_PREEMPT / CMB_RESOURCE_PREEMPT, guards as literal heaps, the holdings of a
stopped process dropped, cmb_random_flip's per-trial cache.

The reference's own fixed-process resource programs - test/test_resource.c (ToolT, model 14), test/test_resourcepool.c
(CheeseT, model 18) and tutorial/tut_2_1.c (Tutorial2T, model 21) - are compiled for the host from the same templates on the
general engine and on the static tier (tests/static_preempt_host.cpp).  The static tier must reproduce, trial for trial, what
the unmodified reference produced: the vectors of tests/golden/cmb_engine_vectors.json with their pop traces, the golden files
test/reference/resource.txt and resourcepool.txt, tutorial 2's vectors, and the live reference build where present.  With too
few spare event slots a trial must be flagged for the general engine, never answered differently."""
import ctypes as C
import json
import random
import re
import struct
import subprocess
import sys
from pathlib import Path

import pytest

from cmb_cases import GOLD, MASTER, RESOURCEPOOL_GOLDEN_LINE, TRACE, case_id, check_trial, inverse_fmix64, wtdsummary_line

ROOT = Path(__file__).resolve().parents[1]
GENERAL, STATIC, ONE_SLOT = 0, 1, 2         # host_preempt_run_trials' engines
CASES = [c for c in GOLD["cases"] if c["model"] in (14, 18)]
TUT2 = json.loads((ROOT / "tests/golden/tutorial2_vectors.json").read_text())
UNIT = {"servers": 1, "num_objects": 0, "arr_mean": (1.0).hex(), "srv_mean": (1.0).hex()}


class HostResult(C.Structure):
    _fields_ = [("events", C.c_uint64), ("objects", C.c_uint64), ("t_end", C.c_double), ("sum_wait", C.c_double),
                ("max_fel", C.c_uint64), ("max_queue", C.c_uint64), ("counter", C.c_uint64 * 8), ("status", C.c_uint32),
                ("pad", C.c_uint32)]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = tmp_path_factory.mktemp("preempt") / "libstatic_preempt_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                    "-shared", "-fPIC", str(ROOT / "tests/static_preempt_host.cpp"), "-o", str(so)], check=True, capture_output=True)
    f = C.CDLL(str(so)).host_preempt_run_trials
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


def _double(u):
    return struct.unpack("<d", struct.pack("<Q", int(u) & (2**64 - 1)))[0]


@pytest.mark.parametrize("case", CASES, ids=case_id)
@pytest.mark.parametrize("engine", [GENERAL, STATIC], ids=["general", "static"])
def test_resource_models_on_the_cpu_match_the_reference_vectors(host, engine, case):
    """Every vector case of models 14 and 18: events, objects, clock, sums, all eight counters, the 2000-pop trace, status 0."""
    n = len(case["trials"])
    out, keys, times = run_host(host, case["model"], engine, case, n)
    for i, want in enumerate(case["trials"]):
        assert out[i].status == 0, (i, out[i].status)
        assert [int(v) for v in out[i].counter] == want["counters8"], (i, "all eight counters")
        check_trial(want, out[i].events, out[i].objects, out[i].t_end, out[i].sum_wait, list(out[i].counter),
                    keys[i * TRACE:(i + 1) * TRACE], times[i * TRACE:(i + 1) * TRACE], f"trial {i}",
                    max_queue=out[i].max_queue if case["model"] == 14 else None)


def test_the_vectors_exercise_what_they_claim(host):
    """The stored trials of model 14 pre-empt (a target loses the resource); model 18's come at two pool sizes."""
    assert sum(t["counters8"][1] > 0 for c in CASES if c["model"] == 14 for t in c["trials"]) >= 3
    assert {c["servers"] for c in CASES if c["model"] == 18} >= {7, 20}


def test_static_tier_reproduces_the_reference_resource_golden_file(host):
    """test/reference/resource.txt on the static tier: history N 30, mean 0.9816, Target_3 pre-empted at t = 6.3280, 85 events."""
    case = {"servers": 1, "num_objects": 25, "arr_mean": (1.0).hex(), "srv_mean": (1.0).hex()}
    out, _, _ = run_host(host, 14, STATIC, case, 1, master=inverse_fmix64(0x34F05C64D7AD598F), trace=0)
    c = list(out[0].counter)
    assert out[0].status == 0 and out[0].events == 85 and out[0].max_queue == 30
    assert "%.4f" % _double(c[3]) == "0.9816" and "%.4f" % _double(c[4]) == "6.3280" and c[5] == 3 and c[1] == 1


def test_static_tier_reproduces_the_reference_resourcepool_golden_file(host):
    """test/reference/resourcepool.txt on the static tier: the reference's seed, 20 units, 100 time units, the file's summary line."""
    import cimba_b200 as cb
    case = {"servers": 20, "num_objects": 100, "arr_mean": (1.0).hex(), "srv_mean": (1.0).hex()}
    out, _, _ = run_host(host, 18, STATIC, case, 1, master=inverse_fmix64(0x34F05C64D7AD598F), trace=0)
    assert out[0].status == 0 and out[0].counter[0] == 120
    assert wtdsummary_line(cb.lib, list(out[0].counter)) == RESOURCEPOOL_GOLDEN_LINE


def test_second_tutorial_on_the_static_tier_matches_the_unmodified_tutorial_source(host):
    """tutorial/tut_2_1.c (about 660 000 events per trial) on the static tier: all 32 vector trials - events, final clock and the
    random stream's next raw output - against the unmodified tutorial source run as a program."""
    n = len(TUT2["trials"])
    out, _, _ = run_host(host, 21, STATIC, UNIT, n, master=TUT2["master"], trace=0)
    for i, want in enumerate(TUT2["trials"]):
        assert out[i].status == 0, i
        assert (out[i].events, float(out[i].t_end).hex(), out[i].counter[0]) == (want["events"], want["t_end"], want["next_raw"]), i


def test_static_equals_general_equals_the_live_reference_on_drawn_parameters(host):
    """Models 14 and 18 at drawn capacities 1..40 and durations: the static tier, the general engine and the live reference build
    (oracle/_ref/librefdrv.so) give the same events, objects, clock, sums and counters for every trial."""
    from oracle_libs import load_ref, run_trials
    ref = load_ref()
    rnd = random.Random(20261015)
    for model in (14, 18):
        for _ in range(4):
            servers = rnd.randint(1, 40)
            nobj = rnd.randint(20, 400)
            case = {"servers": servers, "num_objects": nobj, "arr_mean": (1.0).hex(), "srv_mean": (1.0).hex()}
            first = rnd.randint(0, 5000)
            general, _, _ = run_host(host, model, GENERAL, case, 4, first=first, trace=0)
            static, _, _ = run_host(host, model, STATIC, case, 4, first=first, trace=0)
            want = run_trials(ref, "ref", model, servers, MASTER, first, 4, nobj, 1.0, 1.0, par=0) if ref is not None else None
            for i in range(4):
                row = lambda o: (o.events, o.objects, o.t_end, o.sum_wait, list(o.counter))
                assert static[i].status == 0 and general[i].status == 0, (model, case, i)
                assert row(static[i]) == row(general[i]), (model, case, i)
                if want is not None:
                    assert row(static[i]) == (want[i].events, want[i].objects, want[i].t_end, want[i].sum_wait, list(want[i].counter)), \
                        (model, case, i)
    if ref is None:
        pytest.skip("oracle/_ref/librefdrv.so not built (needs the reference sources): static = general checked only")


def test_too_few_spare_slots_flag_the_trial_and_never_answer_differently(host):
    """One spare event slot where the models want two to eight: each trial is either flagged for the general engine, or its
    answer is the reference's exactly.  Tutorial 2 and the pool test pre-empt several holders at once, so most trials flag."""
    flagged = exact = 0
    n = len(TUT2["trials"])
    out, _, _ = run_host(host, 21, ONE_SLOT, UNIT, n, master=TUT2["master"], trace=0)
    for i, want in enumerate(TUT2["trials"]):
        if out[i].status:
            flagged += 1
        else:
            exact += 1
            assert (out[i].events, float(out[i].t_end).hex(), out[i].counter[0]) == (want["events"], want["t_end"], want["next_raw"]), i
    for case in CASES:
        k = len(case["trials"])
        out, keys, times = run_host(host, case["model"], ONE_SLOT, case, k)
        for i, want in enumerate(case["trials"]):
            if out[i].status:
                flagged += 1
                continue
            exact += 1
            check_trial(want, out[i].events, out[i].objects, out[i].t_end, out[i].sum_wait, list(out[i].counter),
                        keys[i * TRACE:(i + 1) * TRACE], times[i * TRACE:(i + 1) * TRACE], f"trial {i}")
            assert [int(v) for v in out[i].counter] == want["counters8"]
    assert flagged >= n and exact > 0, (flagged, exact)


# ---- registers, stack and spills of the new static-tier instantiations (no GPU needed)
KERNELS = {"ToolT": (4, 2), "CheeseT": (6, 6), "Tutorial2T": (8, 8)}
SRC = """#include "cmb_launch.cuh"
#include "../models/workshop_model.cuh"
#include "../models/cheese_model.cuh"
#include "../models/tutorial2_model.cuh"
namespace cimba_b200 { namespace cmb {
""" + "".join(f"template __global__ void static_trial_kernel<models::{m}, {p}, 0, {e}, {t}>(const StaticArgs);\n"
              for m, (p, e) in KERNELS.items() for t in ("false", "true")) + "}}\n"


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    sys.path.insert(0, str(ROOT))
    import __graft_entry__ as g
    d = tmp_path_factory.mktemp("preempt_resources")
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
    assert re.search(r"\d+ bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", text), text
    assert int(re.search(r"Used (\d+) registers", text).group(1)) <= 255, text
