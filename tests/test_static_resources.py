"""CPU tests of cmb_resourcepool and cmb_resource on the static tier (cimba_b200/csrc/cmb_static.cuh).

examples/repair_model.cuh - a machine shop whose machines share a repair crew (a pool, its usage history on) and an
inspection bench (a resource) - is compiled for the host twice from the same template (tests/static_resources_host.cpp): on
the general engine and on cmb::StaticSim<8, 0>.  Both must reproduce, trial for trial, what the unmodified reference produced
for the same shop written against its own API (tests/golden/repair_vectors.json, and the live build
oracle/_ref/librepairdrv.so where present): events, repairs, clock, downtime, all eight counters and the pop trace.

The static tier has to hand two cases to the general engine, and must say so in the trial's status word: twelve machines
(more processes than its eight slots) and machines that exit while they hold crew (the reference drops their holdings)."""
import ctypes as C
import subprocess
from pathlib import Path

import pytest

from cmb_cases import trace_digest
from repair_cases import GOLD, load_repair_ref, ref_run

ROOT = Path(__file__).resolve().parents[1]
MASTER, TRACE = GOLD["master"], GOLD["trace"]
GENERAL, STATIC = 0, 1              # host_repair_run_trials' engines
PROC_OVERFLOW = 16                  # CIMBA_B200_TRIAL_PROC_OVERFLOW
FALLBACK = ("twelve_machines", "exit_holding")      # the cases the static tier hands to the general engine
CASES = {c["name"]: c for c in GOLD["cases"]}


class HostResult(C.Structure):
    _fields_ = [("events", C.c_uint64), ("objects", C.c_uint64), ("t_end", C.c_double), ("sum_wait", C.c_double),
                ("max_fel", C.c_uint64), ("max_queue", C.c_uint64), ("counter", C.c_uint64 * 8), ("status", C.c_uint32),
                ("pad", C.c_uint32)]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = tmp_path_factory.mktemp("repair") / "libstatic_resources_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                    "-shared", "-fPIC", str(ROOT / "tests/static_resources_host.cpp"), "-o", str(so)], check=True, capture_output=True)
    f = C.CDLL(str(so)).host_repair_run_trials
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double,
                  C.POINTER(C.c_double), C.c_uint32, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double),
                  C.POINTER(HostResult)]
    return f


def run_host(f, model, case, n, first=0, arr=None, srv=None, trace=TRACE):
    out = (HostResult * n)()
    par = (C.c_double * 2)(*case["params"])
    keys = (C.c_uint64 * max(1, n * trace))()
    times = (C.c_double * max(1, n * trace))()
    arr = float.fromhex(case["arr_mean"]) if arr is None else arr
    srv = float.fromhex(case["srv_mean"]) if srv is None else srv
    rc = f(model, case["servers"], MASTER, first, n, case["num_objects"], arr, srv, par, 2, 1 << 26, trace, keys, times, out)
    assert rc == 0
    return out, keys, times


def check(want, o, keys, times, what):
    assert (o.events, o.objects) == (want["events"], want["objects"]), (what, o.events, want["events"])
    assert float(o.t_end).hex() == want["t_end"] and float(o.sum_wait).hex() == want["sum_wait"], what
    assert list(o.counter) == want["counters8"], (what, list(o.counter), want["counters8"])
    assert trace_digest(keys, times, o.events) == want["trace_sha256"], (what, "pop trace")


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("model", [GENERAL, STATIC], ids=["general", "static"])
def test_repair_shop_on_the_cpu_matches_the_reference_vectors(host, model, name):
    case = CASES[name]
    n = len(case["trials"])
    out, keys, times = run_host(host, model, case, n)
    for i, want in enumerate(case["trials"]):
        if model == STATIC and name in FALLBACK:
            # void on the static tier: flagged for the general engine, whose answer is the one above
            assert out[i].status & PROC_OVERFLOW, (name, i, out[i].status)
            continue
        assert out[i].status == 0, (name, i, out[i].status)
        check(want, out[i], keys[i * TRACE:(i + 1) * TRACE], times[i * TRACE:(i + 1) * TRACE], f"{name} trial {i}")


def test_the_vectors_exercise_what_they_claim():
    """Partial grabs in the saturated case, a busy bench everywhere the crew is not deadlocked, the exit before the last
    repair, and a deadlock that ends the trial early."""
    assert all(t["counters8"][0] > 0 for t in CASES["saturated"]["trials"])
    for name, case in CASES.items():
        if name != "deadlock":
            assert all(t["counters8"][1] > 0 for t in case["trials"]), name
            assert all(t["counters8"][7] == 0 and t["counters8"][2] > 0 for t in case["trials"]), name
    machines, cycles = 8, CASES["exit_holding"]["num_objects"]
    assert all(t["objects"] == machines * (cycles - 1) for t in CASES["exit_holding"]["trials"])
    assert all(t["objects"] == 12 * CASES["twelve_machines"]["num_objects"] for t in CASES["twelve_machines"]["trials"])
    assert all(t["objects"] < CASES["deadlock"]["num_objects"] for t in CASES["deadlock"]["trials"])


def test_repair_shop_matches_the_live_reference_build(host):
    """Other trials and parameters than the stored vectors, including a non-unit service mean, against the reference itself."""
    ref = load_repair_ref()
    if ref is None:
        pytest.skip("oracle/_ref/librepairdrv.so not built (needs the reference sources)")
    for servers, nobj, arr, srv, params in ((5, 700, 2.5, 0.37, [8, 0]), (4, 600, 30.0, 3.7, [7, 0]), (2, 900, 11.0, 1.3, [3, 0]),
                                            (1, 500, 4.0, 0.61, [8, 1]), (9, 300, 1.9, 0.93, [16, 0])):
        case = {"servers": servers, "num_objects": nobj, "params": params}
        want = ref_run(ref, servers, MASTER, 11, 5, nobj, arr, srv, params)
        fallback = params[0] > 8 or params[1] != 0
        for model in (GENERAL, STATIC):
            out, _, _ = run_host(host, model, case, 5, first=11, arr=arr, srv=srv, trace=0)
            for i, (o, w) in enumerate(zip(out, want)):
                if model == STATIC and fallback:
                    assert o.status & PROC_OVERFLOW, (params, i)
                    continue
                assert o.status == 0, (model, params, i, o.status)
                assert (o.events, o.objects, o.t_end, o.sum_wait) == (w.events, w.objects, w.t_end, w.sum_wait), (model, params, i)
                assert list(o.counter) == list(w.counter), (model, params, i)
