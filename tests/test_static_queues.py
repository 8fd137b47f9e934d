"""CPU tests of the static tier's cmb_priorityqueue and cmb_condition (cimba_b200/csrc/cmb_static.cuh): the priority queue as a
table scanned under its strict order, handles, position / cancel / reprioritize, the length history, the condition's wait list as
a literal heap with its predicates, its wake-ups in the waiters' own event slots, fel_high for the models that report it.

The reference's own queue programs - test/test_objectqueue.c (GuardedT, models 3 and 11), test/test_priorityqueue.c (model 13) -
and the coverage world QueueAndTideT (model 6) are compiled for the host from the same templates on the general engine and on the
static tier (tests/static_queues_host.cpp).  The static tier must reproduce, trial for trial, what the unmodified reference
produced: the vectors of tests/golden/cmb_engine_vectors.json with their pop traces, the golden files test/reference/objectqueue.txt
and priorityqueue.txt, and the live reference build where present.  A queue beyond the tier's table, or too few spare event slots,
must flag the trial for the general engine, never answer differently.  A small model of the host file's own runs the tier's first
form (no static_interrupts) with both containers."""
import ctypes as C
import json
import random
import re
import subprocess
import sys
from pathlib import Path

import pytest

from cmb_cases import GOLD, MASTER, TRACE, case_id, check_trial, inverse_fmix64

ROOT = Path(__file__).resolve().parents[1]
GENERAL, STATIC, ONE_SLOT = 0, 1, 2         # host_queues_run_trials' engines
TWO_CLASS = 100                             # the host file's first-form model
MODELS = (3, 6, 11, 13)
CASES = [c for c in GOLD["cases"] if c["model"] in MODELS]
KAT_SEED = 0x34F05C64D7AD598F


class HostResult(C.Structure):
    _fields_ = [("events", C.c_uint64), ("objects", C.c_uint64), ("t_end", C.c_double), ("sum_wait", C.c_double),
                ("max_fel", C.c_uint64), ("max_queue", C.c_uint64), ("counter", C.c_uint64 * 8), ("status", C.c_uint32),
                ("pad", C.c_uint32)]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = tmp_path_factory.mktemp("queues") / "libstatic_queues_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                    "-shared", "-fPIC", str(ROOT / "tests/static_queues_host.cpp"), "-o", str(so)], check=True, capture_output=True)
    f = C.CDLL(str(so)).host_queues_run_trials
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


@pytest.mark.parametrize("case", CASES, ids=case_id)
@pytest.mark.parametrize("engine", [GENERAL, STATIC], ids=["general", "static"])
def test_queue_models_on_the_cpu_match_the_reference_vectors(host, engine, case):
    """Every vector case of models 3, 6, 11 and 13: events, objects, clock, sums, all eight counters, max_queue (the history's
    size for 11 and 13, fel_high for 3 and 6), the 2000-pop trace, status 0."""
    n = len(case["trials"])
    out, keys, times = run_host(host, case["model"], engine, case, n)
    for i, want in enumerate(case["trials"]):
        assert out[i].status == 0, (i, out[i].status)
        assert [int(v) for v in out[i].counter] == want["counters8"], (i, "all eight counters")
        check_trial(want, out[i].events, out[i].objects, out[i].t_end, out[i].sum_wait, list(out[i].counter),
                    keys[i * TRACE:(i + 1) * TRACE], times[i * TRACE:(i + 1) * TRACE], f"trial {i}",
                    max_queue=out[i].max_queue if case["model"] in (11, 13) else None)
        if case["model"] in (3, 6):
            assert out[i].max_queue == want["max_fel"], (i, "fel_high")


def test_the_vectors_exercise_what_they_claim(host):
    """The stored trials of model 6 reposition, cancel and reprioritize by handle and wake the condition's waiters; the guarded
    queue tests come at capacities 2 and 3 as well as 10 (both guards in play)."""
    six = [t for c in CASES if c["model"] == 6 for t in c["trials"]]
    assert all(t["counters8"][3] > 1000 and t["counters8"][4] > 0 and t["counters8"][5] > 0 for t in six)
    assert {c["servers"] for c in CASES} >= {2, 3, 10}


@pytest.mark.parametrize("model", [11, 13])
def test_static_tier_reproduces_the_reference_queue_golden_files(host, model):
    """test/reference/objectqueue.txt (model 11) and priorityqueue.txt (model 13) on the static tier: the reference's seed, capacity
    10, 10^6 time units: length history N 5689021, time-weighted mean 5.008, and every word equal to the reference's record."""
    import struct
    gold = json.loads((ROOT / "tests/golden/reference_vectors.json").read_text())
    want = [t for t in gold["trials"] if t["model"] == model and t["num_objects"] == 1_000_000][0]
    case = {"servers": 10, "num_objects": 1_000_000, "arr_mean": (1.0).hex(), "srv_mean": (1.0).hex()}
    out, _, _ = run_host(host, model, STATIC, case, 1, master=inverse_fmix64(KAT_SEED), trace=0)
    o = out[0]
    mean = struct.unpack("<d", struct.pack("<Q", o.counter[6]))[0]
    assert o.status == 0 and o.max_queue == 5689021 and "%.4g" % mean == "5.008"
    assert list(o.counter) == want["counters"]
    assert (o.events, o.objects, float(o.t_end).hex(), float(o.sum_wait).hex()) == \
           (want["events"], want["objects"], want["t_end"], want["sum_wait"])


def test_static_equals_general_equals_the_live_reference_on_drawn_parameters(host):
    """Models 3, 6, 11 and 13 at drawn capacities 1..16 and durations: the static tier, the general engine and the live reference
    build (oracle/_ref/librefdrv.so) give the same events, objects, clock, sums and counters for every trial."""
    from oracle_libs import load_ref, run_trials
    ref = load_ref()
    rnd = random.Random(20261016)
    for model in MODELS:
        for _ in range(4):
            servers = rnd.randint(1, 16)
            nobj = rnd.randint(100, 1500)
            arr, srv = rnd.choice([0.5, 0.8, 1.0, 1.6]), rnd.choice([0.6, 1.0, 1.4])
            case = {"servers": servers, "num_objects": nobj, "arr_mean": float(arr).hex(), "srv_mean": float(srv).hex()}
            first = rnd.randint(0, 5000)
            general, _, _ = run_host(host, model, GENERAL, case, 4, first=first, trace=0)
            static, _, _ = run_host(host, model, STATIC, case, 4, first=first, trace=0)
            want = run_trials(ref, "ref", model, servers, MASTER, first, 4, nobj, arr, srv, par=0) if ref is not None else None
            for i in range(4):
                assert static[i].status == 0 and general[i].status == 0, (model, case, i, static[i].status)
                assert row(static[i]) == row(general[i]), (model, case, i)
                if want is not None:
                    got = (static[i].events, static[i].objects, static[i].t_end, static[i].sum_wait, list(static[i].counter))
                    assert got == (want[i].events, want[i].objects, want[i].t_end, want[i].sum_wait, list(want[i].counter)), \
                        (model, case, i)
    if ref is None:
        pytest.skip("oracle/_ref/librefdrv.so not built (needs the reference sources): static = general checked only")


def test_a_queue_above_the_table_or_the_window_flags_the_trial_and_never_answers_differently(host):
    """Capacity 40: the priority queue can outgrow its 16-entry table (models 6 and 13) and the object queue its 32-entry window
    (models 3 and 11, which have no HBM ring on this route).  Each trial is either flagged for the general engine with the
    queue-overflow bit, or equal to the general engine's; and the heavy-traffic runs flag some."""
    flagged = exact = 0
    for model in MODELS:
        case = {"servers": 40, "num_objects": 3000, "arr_mean": (0.5).hex(), "srv_mean": (1.0).hex()}
        general, _, _ = run_host(host, model, GENERAL, case, 24, first=100, trace=0)
        static, _, _ = run_host(host, model, STATIC, case, 24, first=100, trace=0)
        for i in range(24):
            assert general[i].status == 0
            if static[i].status:
                assert static[i].status == 1, (model, i, static[i].status)   # CIMBA_B200_TRIAL_QUEUE_OVERFLOW
                flagged += 1
            else:
                exact += 1
                assert row(static[i]) == row(general[i]), (model, i)
    assert flagged > 0, (flagged, exact)


def test_one_spare_slot_too_few_flags_the_trial_and_never_answers_differently(host):
    """One spare event slot where the models want two (the end event and an interrupt): each trial is either flagged, or its
    answer is the reference's exactly - and a trial with an interrupt flags."""
    flagged = exact = 0
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
    assert flagged > 0, (flagged, exact)


def test_first_form_two_class_queue_with_an_observer_matches_the_general_engine(host):
    """The tier's first form (no static_interrupts): a two-class priority M/M/1 and an observer waiting on a condition, 300 trials
    at drawn loads, capacities and lengths - static equals general in every word, and the queue and condition are exercised."""
    rnd = random.Random(31)
    total_hits = total_passes = 0
    for _ in range(6):
        case = {"servers": rnd.randint(3, 16), "num_objects": rnd.randint(50, 800), "arr_mean": rnd.choice([0.8, 1.0, 1.25]).hex(),
                "srv_mean": rnd.choice([0.7, 1.0]).hex()}
        first = rnd.randint(0, 10_000)
        general, gk, gt = run_host(host, TWO_CLASS, GENERAL, case, 50, first=first)
        static, sk, st = run_host(host, TWO_CLASS, STATIC, case, 50, first=first)
        for i in range(50):
            assert general[i].status == 0 and static[i].status == 0, (case, i, static[i].status)
            assert row(static[i]) == row(general[i]), (case, i)
            n = min(int(general[i].events), TRACE)
            assert list(gk[i * TRACE:i * TRACE + n]) == list(sk[i * TRACE:i * TRACE + n]), (case, i)
            assert list(gt[i * TRACE:i * TRACE + n]) == list(st[i * TRACE:i * TRACE + n]), (case, i)
            total_hits += static[i].counter[4]
            total_passes += static[i].counter[5]
    assert total_hits > 0 and total_passes > 0


# ---- registers, stack and spills of the new static-tier instantiations (no GPU needed)
KERNELS = {"GuardedQueueT": (7, 1), "GuardedRecordedQueueT": (7, 1), "GuardedPriorityQueueT": (7, 0), "QueueAndTideT": (8, 0)}
SRC = """#include "cmb_launch.cuh"
#include "../models/guarded_model.cuh"
#include "../models/coverage_models.cuh"
namespace cimba_b200 { namespace cmb {
""" + "".join(f"template __global__ void static_trial_kernel<models::{m}, {p}, {q}, 2, {t}>(const StaticArgs);\n"
              for m, (p, q) in KERNELS.items() for t in ("false", "true")) + "}}\n"


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    sys.path.insert(0, str(ROOT))
    import __graft_entry__ as g
    d = tmp_path_factory.mktemp("queue_resources")
    (d / "k.cu").write_text(SRC)
    flags = [f for f in g.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    cmd = [g._nvcc(), *flags, "-Xptxas", "-v", "-I", str(g.CSRC), "-I", str(ROOT / "include"), "-cubin", "-o", str(d / "k.cubin"),
           str(d / "k.cu")]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    report = {}
    for m in re.finditer(r"Compiling entry function '\w*static_trial_kernelINS_6models\d+(\w+?)ELi\d+ELi\d+ELi2ELb([01])E\w*' "
                         r"for 'sm_90a'\n(.*?)(?=ptxas info\s+: Compile time)", p.stderr, re.S):
        report[(m.group(1), m.group(2) == "1")] = m.group(3)
    assert set(report) == {(m, t) for m in KERNELS for t in (False, True)}, p.stderr
    return report


@pytest.mark.parametrize("trace", [False, True])
@pytest.mark.parametrize("model", list(KERNELS))
def test_new_instantiations_build_without_spills(ptxas_report, model, trace):
    """The control block may live on the stack (the guard heaps and the queue table are indexed at run time); nothing may spill."""
    text = ptxas_report[(model, trace)]
    stack = re.search(r"(\d+) bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", text)
    regs = re.search(r"Used (\d+) registers", text)
    assert stack and regs and int(regs.group(1)) <= 255, text
    print(f"{model} trace={trace}: {regs.group(1)} registers, {stack.group(1)} bytes stack")
