"""CPU tests of the static tier's timers, resume / yield, waits on processes and events, the model's events by handle and observers
(cimba_b200/csrc/cmb_static.cuh, the second form with static_waits).

The coverage world FrontDeskT (model 8: timers added, cancelled, set and cleared, yield + resume, wait_process on a clerk that exits
and is started again, wait_event on bells that get rescheduled, reprioritized and cancelled, a condition whose guard observes the
desk's guard) is compiled for the host from one template on the general engine and on the static tier (tests/static_timers_host.cpp).
The static tier must reproduce, trial for trial, what the unmodified reference produced: the vectors of
tests/golden/cmb_engine_vectors.json with their pop traces, and the live reference build where present.  With one spare event slot
too few it must flag the trial for the general engine, never answer differently.  A small model of the host file's own - customers
whose patience timers run out during partial grabs of a pool, and a dispatcher that resumes the yielded ones - checks the tier
against the general engine word for word, and in the tier's first form, where a timer must send the trial to the general engine."""
import ctypes as C
import random
import re
import subprocess
import sys
from pathlib import Path

import pytest

from cmb_cases import GOLD, MASTER, TRACE, case_id, check_trial

ROOT = Path(__file__).resolve().parents[1]
GENERAL, STATIC, ONE_SLOT, FIRST_FORM = 0, 1, 2, 3     # host_timers_run_trials' engines
FRONT_DESK, PATIENCE = 8, 200                           # model 8 and the host file's own model
CASES = [c for c in GOLD["cases"] if c["model"] == FRONT_DESK]
PROC_OVERFLOW = 16                                      # CIMBA_B200_TRIAL_PROC_OVERFLOW


class HostResult(C.Structure):
    _fields_ = [("events", C.c_uint64), ("objects", C.c_uint64), ("t_end", C.c_double), ("sum_wait", C.c_double),
                ("max_fel", C.c_uint64), ("max_queue", C.c_uint64), ("counter", C.c_uint64 * 8), ("status", C.c_uint32),
                ("pad", C.c_uint32)]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = tmp_path_factory.mktemp("timers") / "libstatic_timers_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                    "-shared", "-fPIC", str(ROOT / "tests/static_timers_host.cpp"), "-o", str(so)], check=True, capture_output=True)
    lib = C.CDLL(str(so))
    f = lib.host_timers_run_trials
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


def drawn_case(rnd, servers=1):
    return {"servers": servers, "num_objects": rnd.randint(50, 1500), "arr_mean": rnd.choice([0.4, 0.8, 1.0, 2.0]).hex(),
            "srv_mean": rnd.choice([0.3, 0.6, 1.0, 1.2]).hex()}


@pytest.mark.parametrize("case", CASES, ids=case_id)
@pytest.mark.parametrize("engine", [GENERAL, STATIC], ids=["general", "static"])
def test_front_desk_on_the_cpu_matches_the_reference_vectors(host, engine, case):
    """Every vector case of model 8: events, objects, clock, sums, all eight counters, fel_high, the 2000-pop trace, status 0."""
    n = len(case["trials"])
    out, keys, times = run_host(host, FRONT_DESK, engine, case, n)
    for i, want in enumerate(case["trials"]):
        assert out[i].status == 0, (i, out[i].status)
        assert [int(v) for v in out[i].counter] == want["counters8"], (i, "all eight counters")
        check_trial(want, out[i].events, out[i].objects, out[i].t_end, out[i].sum_wait, list(out[i].counter),
                    keys[i * TRACE:(i + 1) * TRACE], times[i * TRACE:(i + 1) * TRACE], f"trial {i}")
        assert out[i].max_queue == want["max_fel"], (i, "fel_high")


def test_the_vectors_exercise_what_they_claim():
    """The stored trials of model 8 time out, restart the clerk, reschedule, reprioritize and cancel the bell, and wake the
    observer's waiter."""
    c = [sum(t["counters8"][k] for c in CASES for t in c["trials"]) for k in range(8)]
    assert c[1] > 0 and c[2] > 0 and c[3] > 0 and c[4] > 0 and c[5] >= 10101 and c[6] >= 1001, c


def test_static_equals_general_equals_the_live_reference_on_drawn_parameters(host):
    """Model 8 at drawn durations and means: the static tier, the general engine and the live reference build
    (oracle/_ref/librefdrv.so) give the same events, objects, clock, sums, counters and fel_high for every trial."""
    from oracle_libs import load_ref, run_trials
    ref = load_ref()
    rnd = random.Random(20261016)
    for _ in range(6):
        case = drawn_case(rnd)
        first = rnd.randint(0, 5000)
        general, _, _ = run_host(host, FRONT_DESK, GENERAL, case, 8, first=first, trace=0)
        static, _, _ = run_host(host, FRONT_DESK, STATIC, case, 8, first=first, trace=0)
        arr, srv = float.fromhex(case["arr_mean"]), float.fromhex(case["srv_mean"])
        want = run_trials(ref, "ref", FRONT_DESK, 1, MASTER, first, 8, case["num_objects"], arr, srv, par=0) if ref is not None else None
        for i in range(8):
            assert static[i].status == 0 and general[i].status == 0, (case, i, static[i].status)
            assert row(static[i]) == row(general[i]), (case, i)
            if want is not None:
                got = (static[i].events, static[i].objects, static[i].t_end, static[i].sum_wait, list(static[i].counter),
                       static[i].max_queue)
                assert got == (want[i].events, want[i].objects, want[i].t_end, want[i].sum_wait, list(want[i].counter),
                               want[i].max_fel), (case, i)
    if ref is None:
        pytest.skip("oracle/_ref/librefdrv.so not built (needs the reference sources): static = general checked only")


def test_one_spare_slot_too_few_flags_the_trial_and_never_answers_differently(host):
    """One spare event slot fewer than the route gives model 8: each vector trial is either flagged, or its answer is the
    reference's exactly - and some flag."""
    flagged = exact = 0
    for case in CASES:
        k = len(case["trials"])
        out, keys, times = run_host(host, FRONT_DESK, ONE_SLOT, case, k)
        for i, want in enumerate(case["trials"]):
            if out[i].status:
                flagged += 1
                continue
            exact += 1
            check_trial(want, out[i].events, out[i].objects, out[i].t_end, out[i].sum_wait, list(out[i].counter),
                        keys[i * TRACE:(i + 1) * TRACE], times[i * TRACE:(i + 1) * TRACE], f"trial {i}")
            assert out[i].max_queue == want["max_fel"]
    assert flagged > 0, (flagged, exact)


def test_patience_timers_and_resumes_match_the_general_engine(host):
    """The host file's model on a 2-unit pool: 300 trials at drawn lengths and means, static equals general in every word and
    in the pop traces; timeouts, timeouts that roll back a partial grab, resumes by the dispatcher and timers that let a yielded
    customer go on alone all happen."""
    rnd = random.Random(77)
    total = [0] * 8
    for _ in range(6):
        case = drawn_case(rnd, servers=2)
        case["num_objects"] = rnd.randint(20, 400)
        first = rnd.randint(0, 10_000) | 1
        general, gk, gt = run_host(host, PATIENCE, GENERAL, case, 50, first=first)
        static, sk, st = run_host(host, PATIENCE, STATIC, case, 50, first=first)
        for i in range(50):
            assert general[i].status == 0 and static[i].status == 0, (case, i, static[i].status)
            assert row(static[i]) == row(general[i]), (case, i)
            n = min(int(general[i].events), TRACE)
            assert list(gk[i * TRACE:i * TRACE + n]) == list(sk[i * TRACE:i * TRACE + n]), (case, i)
            assert list(gt[i * TRACE:i * TRACE + n]) == list(st[i * TRACE:i * TRACE + n]), (case, i)
            for k in range(8):
                total[k] += static[i].counter[k]
    served, timeouts, rolled_back, resumed, alone, resumes, cancelled, _ = total
    assert served > 0 and timeouts > 0 and rolled_back > 0 and resumed > 0 and alone > 0 and cancelled > 0, total
    assert resumes >= resumed


def test_first_form_flags_every_trial_that_reaches_a_timer(host):
    """The same model in the tier's first form (no static_interrupts), where timers do not exist: a trial is either flagged for
    the general engine or equal to it word for word; every trial with a served or timed-out customer (so a timer) is flagged, and
    the short trials without an arrival are answered exactly."""
    flagged = exact = 0
    for nobj, arr in ((1, 50.0), (2, 30.0), (300, 1.0)):
        case = {"servers": 2, "num_objects": nobj, "arr_mean": arr.hex(), "srv_mean": (1.0).hex()}
        general, _, _ = run_host(host, PATIENCE, GENERAL, case, 64, first=9, trace=0)
        first_form, _, _ = run_host(host, PATIENCE, FIRST_FORM, case, 64, first=9, trace=0)
        for i in range(64):
            assert general[i].status == 0
            if general[i].counter[0] + general[i].counter[1] > 0:
                assert first_form[i].status & PROC_OVERFLOW, (case, i)
            if first_form[i].status:
                flagged += 1
            else:
                exact += 1
                assert row(first_form[i]) == row(general[i]), (case, i)
    assert flagged > 0 and exact > 0, (flagged, exact)


# ---- registers, stack and spills of the new static-tier instantiations (no GPU needed)
SRC = """#include "cmb_launch.cuh"
#include "../models/coverage_models.cuh"
namespace cimba_b200 { namespace cmb {
""" + "".join(f"template __global__ void static_trial_kernel<models::FrontDeskT, 8, 0, models::FRONTDESK_SPARE_SLOTS, {t}>"
              f"(const StaticArgs);\n" for t in ("false", "true")) + "}}\n"


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    sys.path.insert(0, str(ROOT))
    import __graft_entry__ as g
    d = tmp_path_factory.mktemp("timer_resources")
    (d / "k.cu").write_text(SRC)
    flags = [f for f in g.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    cmd = [g._nvcc(), *flags, "-Xptxas", "-v", "-I", str(g.CSRC), "-I", str(ROOT / "include"), "-cubin", "-o", str(d / "k.cubin"),
           str(d / "k.cu")]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    report = {}
    for m in re.finditer(r"Compiling entry function '\w*static_trial_kernelINS_6models10FrontDeskTELi8ELi0ELi\d+ELb([01])E\w*' "
                         r"for 'sm_90a'\n(.*?)(?=ptxas info\s+: Compile time)", p.stderr, re.S):
        report[m.group(1) == "1"] = m.group(2)
    assert set(report) == {False, True}, p.stderr
    return report


@pytest.mark.parametrize("trace", [False, True])
def test_front_desk_kernel_builds_without_spills(ptxas_report, trace):
    """The control block may live on the stack (the guard heaps and the observer links are reached by address); nothing may
    spill."""
    text = ptxas_report[trace]
    stack = re.search(r"(\d+) bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", text)
    regs = re.search(r"Used (\d+) registers", text)
    assert stack and regs and int(regs.group(1)) <= 255, text
    print(f"FrontDeskT trace={trace}: {regs.group(1)} registers, {stack.group(1)} bytes stack")
