"""CPU tests of the event list used as a whole - cmb_event_queue_initialize / _is_empty / _count / _clear, cmb_event_time /
_priority and cmb_event_pattern_find / _count / _cancel with the CMB_ANY_* wildcards - on both engines' source text compiled for
the CPU (tests/event_queue_host.cpp): the general engine (cmb::Sim) and the static tier's second form with events by handle.

examples/event_model.cuh's EventTestT is the reference's own event-queue test (test/test_event.c) as model code.  On the general
engine its notes print the reference's text, event-list dumps read from the heap array: byte for byte the golden file
test/reference/event.txt (tests/golden/event.txt) at its seed, and the unmodified test program's output (oracle/_ref/test_event)
at 32 more seeds.  Its rows and pop traces equal tests/golden/event_vectors.json (the unmodified reference library,
oracle/ref_build/event_driver.c).  On the static tier it is flagged at the wildcard loop's first find (three matches, whose order
only the heap array decides) and the re-run prints the same text.  EventChurnT is answered by the static tier without a flag,
row for row and trace for trace as the general engine, at 1000 seeds.  EdgeT (this file's host build) pins the corners."""
import ctypes as C
import struct
import subprocess
from pathlib import Path

import pytest

from event_cases import GOLDEN_SEED, MASTER, TRACE_CAP, fmix64, load_event_ref, ref_run, vectors
from oracle_libs import Result

ROOT = Path(__file__).resolve().parents[1]
PROC_OVERFLOW, BAD_ARGUMENT = 16, 128
TEST_MODEL, CHURN_MODEL, EDGE_MODEL = 0, 1, 2
GENERAL, STATIC = 0, 1


class HostResult(C.Structure):
    _fields_ = Result._fields_ + [("status", C.c_uint32), ("pad", C.c_uint32)]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = tmp_path_factory.mktemp("event_queue") / "libevent_queue_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", str(ROOT / "tests/event_queue_host.cpp"),
                    "-o", str(so)], check=True, capture_output=True)
    lib = C.CDLL(str(so))
    lib.host_event_test_text.restype = C.c_uint32
    lib.host_event_test_text.argtypes = [C.c_int, C.c_uint64, C.c_char_p, C.c_uint64, C.POINTER(C.c_uint32)]
    lib.host_event_run_trials.restype = C.c_int
    lib.host_event_run_trials.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double,
                                          C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double), C.POINTER(HostResult)]
    lib.host_event_any_subject.restype = C.c_uint32
    return lib


def text(lib, engine, seed):
    """(text, status, flag point) of EventTestT at `seed`; engine 1 = the static tier, re-run on the general engine if flagged."""
    buf = C.create_string_buffer(1 << 16)
    point = C.c_uint32(0)
    status = lib.host_event_test_text(engine, seed, buf, len(buf), C.byref(point))
    return buf.value.decode(), status, point.value


def run(lib, model, engine, count, first=0, master=MASTER, num_objects=40, srv_mean=0.8, param=0.0, cap=0):
    """[(status, events, objects, t_end hex, counters, trace)] of trials [first, first + count)."""
    out = (HostResult * count)()
    keys = (C.c_uint64 * max(count * cap, 1))()
    times = (C.c_double * max(count * cap, 1))()
    assert lib.host_event_run_trials(model, engine, master, first, count, num_objects, srv_mean, param, cap, keys, times, out) == 0
    rows = []
    for i, r in enumerate(out):
        n = min(r.events, cap)
        trace = [(keys[i * cap + k], float(times[i * cap + k]).hex()) for k in range(n)]
        rows.append((r.status, r.events, r.objects, float(r.t_end).hex(), list(r.counter), trace))
    return rows


def test_golden_text_on_the_general_engine(host):
    """test/reference/event.txt byte for byte: every dump in heap-array order, the found event, the cancels and the run's log."""
    got, status, _ = text(host, GENERAL, GOLDEN_SEED)
    assert status == 0
    assert got == (ROOT / "tests/golden/event.txt").read_text()


@pytest.mark.skipif(not (ROOT / "oracle/_ref/test_event").exists(), reason="oracle/_ref/test_event not built (no reference sources)")
def test_text_equals_the_unmodified_reference_program(host):
    """oracle/_ref/test_event -s <seed> (test/test_event.c compiled unmodified) at 32 more seeds."""
    for i in range(1, 33):
        seed = fmix64(MASTER, i)
        want = subprocess.run([str(ROOT / "oracle/_ref/test_event"), "-s", hex(seed)], check=True, capture_output=True).stdout.decode()
        got, status, _ = text(host, GENERAL, seed)
        assert status == 0 and got == want, (i, hex(seed))


@pytest.mark.parametrize("trial", [0, 1, 2, 7, 21, 63])
def test_static_tier_flags_the_test_at_its_first_multi_match_find(host, trial):
    """Not flagged through the first dump after the single-match find and cancel; flagged at the wildcard loop (dump 2); the
    re-run's text is the general engine's."""
    seed = fmix64(MASTER, trial)
    got, status, point = text(host, STATIC, seed)
    assert status & PROC_OVERFLOW and point == 2, (trial, status, point)
    want, _, _ = text(host, GENERAL, seed)
    assert got == want
    if trial == 0:
        assert got == (ROOT / "tests/golden/event.txt").read_text()


def test_vectors_on_the_general_engine(host):
    """The 64 stored trials: events, clock, the eight counters and the whole pop trace; the static tier flags every one."""
    want = vectors()
    assert want["master"] == MASTER
    n = len(want["trials"])
    got = run(host, TEST_MODEL, GENERAL, n, cap=TRACE_CAP)
    for i, (w, g) in enumerate(zip(want["trials"], got)):
        assert w["seed"] == fmix64(MASTER, i)
        assert g[:2] == (0, w["events"]) and g[3] == w["t_end"] and g[4] == w["counters"], i
        assert g[5] == [tuple(x) for x in w["trace"]], i
    assert all(s & PROC_OVERFLOW for s, *_ in run(host, TEST_MODEL, STATIC, n))


@pytest.mark.skipif(load_event_ref() is None, reason="oracle/_ref/libeventdrv.so not built (no reference sources)")
def test_vectors_equal_the_live_reference_driver():
    lib = load_event_ref()
    want = vectors()["trials"]
    for w, (r, keys, times) in zip(want, ref_run(lib, MASTER, 0, len(want))):
        assert (r.events, float(r.t_end).hex(), list(r.counter)) == (w["events"], w["t_end"], w["counters"])
        assert [[k, float(t).hex()] for k, t in zip(keys, times)] == w["trace"]


def test_churn_static_equals_general_without_a_flag(host):
    """EventChurnT at 1000 seeds: rows and pop traces identical, status 0 on both, and the queries did real work."""
    cap = 1024
    general = run(host, CHURN_MODEL, GENERAL, 1000, cap=cap)
    static = run(host, CHURN_MODEL, STATIC, 1000, cap=cap)
    assert all(r[0] == 0 for r in general) and all(r[0] == 0 for r in static)
    assert all(r[1] < cap for r in general)
    assert static == general
    assert sum(r[4][6] for r in general) > 1000                    # blips cancelled by pattern
    assert all(r[4][1] == 1 for r in general)                      # empty only after the end event's clear
    assert any(r[4][4] % 1000 > 0 for r in general)                # blips were counted


def _f(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


@pytest.mark.parametrize("engine", [GENERAL, STATIC])
def test_edge_cases(host, engine):
    (s0, _, _, _, c0, _), = run(host, EDGE_MODEL, engine, 1, param=0.0)
    assert s0 == BAD_ARGUMENT and c0[2] == BAD_ARGUMENT                 # time / priority of a cancelled handle
    assert _f(c0[0]) == 0.0 and c0[1] == 0                              # ... return 0
    assert _f(c0[3]) == 7.0 and c0[4] == (1 << 64) - 4                  # a live one: its time and priority

    (s1, _, _, _, c1, _), = run(host, EDGE_MODEL, engine, 1, param=1.0)
    assert s1 == 0
    assert c1[:4] == [0, 0, 0, 2]           # two process starts pending: no pattern sees them, subject 0 / 1 included
    assert c1[4:7] == [1, 1, 21]            # a model event of subject 0: found, then cancelled by wildcard; the starts stay

    (s2, _, _, _, c2, _), = run(host, EDGE_MODEL, engine, 1, param=2.0)
    assert s2 == 0 and c2[:6] == [1, 2, 1, 1, 1, 0]                     # CMB_ANY_SUBJECT is not NIL
    assert host.host_event_any_subject() != 0xFFFFFFFF

    (s3, _, _, _, c3, _), = run(host, EDGE_MODEL, engine, 1, param=3.0)
    assert s3 == 0
    assert c3[1] == 3 and c3[2] == 10       # after the clear: count 0, empty; cmb_event_current() is the clearing event
    assert c3[3] == 0                       # the awaited handle: not scheduled, cancel false
    assert c3[4] == 4                       # keys run on: awaited 1, start 2, clear 3, the next 4
    assert c3[5] == 1 and c3[7] == 0        # the waiter still running, never woken; nothing else pending

    (s4, _, _, _, c4, _), = run(host, EDGE_MODEL, engine, 1, param=4.0)
    assert s4 == BAD_ARGUMENT and c4[1] == 0                            # initialize before any schedule: fine ...
    assert _f(c4[0]) == 2.0 and _f(c4[2]) == 2.0                        # ... after one: flagged, the clock stays
