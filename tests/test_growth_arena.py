"""The general engine's growth arena (cmb::Arena, cimba_b200/csrc/cmb_device.cuh) at its edges, on the CPU: the engine's host build
(tests/cmb_engine_host.cpp) compiled with AddressSanitizer and UndefinedBehaviorSanitizer runs, for every model it builds, a shape
that grows the model's containers, with the arena a trial needs, one 16-byte step less, half of it, 4 KB and 1 GB.

A trial's need is the arena cursor when it ends (host_cmb_run_trials_used).  Allocation order is fixed by the seed, so a trial
must be flagged (CIMBA_B200_TRIAL_ARENA_EXHAUSTED) exactly when its arena is smaller than that, must then end promptly without a
stray write, and must otherwise give the same result as with 1 GB - the reference's answer where a golden vector exists.

The GPU test of the same path (tests/test_gpu_growth_arena.py) runs experiment-scale jobs whose trials need more arena than their
route asks for; here each of those shapes is checked on a strided sample of its trials to need at least twice that arena."""
import ctypes as C
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))

from arena_cases import GPU_SHAPES, MASTER, SAMPLE, SAMPLED_NEED, estimated_need, need_key, rings_bytes, sample_trials, shape_of  # noqa: E402
from cmb_cases import GOLD, case_id, check_trial  # noqa: E402

ARENA_EXHAUSTED = 64            # CIMBA_B200_TRIAL_ARENA_EXHAUSTED (the worker runs without the package)
BIG = 1 << 30
CALL_SECONDS = 120              # no single call may take longer: a trial that runs out of arena must end, not spin
BISECTED = 2                    # trials per shape whose need is also found by bisection


def _gold(cid):
    return next(c for c in GOLD["cases"] if case_id(c) == cid)


def _case(model, servers, num_objects, arr_mean, srv_mean=1.0, params=(), trials=4):
    return {"model": model, "servers": servers, "num_objects": num_objects, "arr_mean": float(arr_mean).hex(),
            "srv_mean": float(srv_mean).hex(), "params": list(params), "trials": [None] * trials}


# One shape per model of the host build that grows its containers: a golden case where one does, otherwise drawn here.
SHAPES = {
    "mm1-overload":      _gold("model0-s1-n20000-a0.952"),
    "gg1-overload":      _case(1, 1, 20_000, 1 / 1.05),
    "mm1rec-overload":   _case(9, 1, 20_000, 1 / 1.05),
    "mmc8-overload":     _gold("model2-s8-n20000-a0.119"),
    "mmc64-overload":    _case(2, 64, 5_000, 1 / (64 * 1.25)),
    "renege-1000":       _gold("model16-s1000-n60-a4.000"),
    "harbor":            _gold("model10-s10-n1500-a2.000"),
    "park":              _case(20, 1, 0, 1.0, trials=3),
    "hold-2000":         _gold("model7-s2000-n6-a1.000"),
    "cheese":            _gold("model18-s7-n300-a1.000"),
    "tutorial1":         _gold("model19-s1-n20000-a1.111"),
    "tutorial2":         _case(21, 1, 0, 1.0, trials=2),
    "guarded":           _gold("model3-s10-n3000-a1.000"),
    "guarded-recorded":  _gold("model11-s10-n20000-a1.000"),
    "prioq-recorded":    _gold("model13-s3-n3000-a0.700"),
    "workshop":          _gold("model5-s10-n3000-a1.000"),
    "workshop-recorded": _gold("model12-s10-n10000-a1.000"),
    "prioq":             _gold("model6-s6-n3000-a0.700"),
    "timers":            _gold("model8-s1-n3000-a1.000"),
    "preempt":           _gold("model4-s8-n3000-a1.000"),
    "tool":              _gold("model14-s1-n5000-a1.000"),
    "tandem":            _gold("model17-s4-n20000-a1.300"),
}


# ------------------------------------------------------------------------------------------------ the worker (a subprocess)
class HostResult(C.Structure):
    _fields_ = [("events", C.c_uint64), ("objects", C.c_uint64), ("t_end", C.c_double), ("sum_wait", C.c_double),
                ("max_fel", C.c_uint64), ("max_queue", C.c_uint64), ("counter", C.c_uint64 * 8), ("status", C.c_uint32),
                ("pad", C.c_uint32)]


def _worker(so, job):
    """Runs in a subprocess with the sanitizer runtime preloaded; prints one JSON line"""
    f = C.CDLL(so).host_cmb_run_trials_used
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double,
                  C.POINTER(C.c_double), C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(HostResult),
                  C.POINTER(C.c_uint64)]
    c = job["case"]
    par = (C.c_double * max(1, len(c["params"])))(*c["params"])
    slowest = 0.0

    def run(firsts, arena):
        nonlocal slowest
        rows, used = [], []
        for first in firsts:            # one call per trial: each trial has the whole arena to itself
            out, u = (HostResult * 1)(), (C.c_uint64 * 1)()
            t = time.monotonic()
            assert f(c["model"], c["servers"], job["master"], first, 1, c["num_objects"], float.fromhex(c["arr_mean"]),
                     float.fromhex(c["srv_mean"]), par, len(c["params"]), arena, 0, None, None, out, u) == 0
            slowest = max(slowest, time.monotonic() - t)
            o = out[0]
            rows.append([o.events, o.objects, o.t_end.hex(), o.sum_wait.hex(), o.max_fel, o.max_queue, list(o.counter), o.status])
            used.append(u[0])
        return rows, used

    trials = job["trials"]
    if job["kind"] == "need":           # the GPU shapes' sample: needs only
        rows, used = run(trials, 1 << 28)
        print(json.dumps({"need": used, "status": [r[7] for r in rows], "slowest": slowest}))
        return
    big, need = run(trials, BIG)
    at = {}
    for k, t in enumerate(trials):
        for arena in sorted({need[k], need[k] - 16, need[k] // 2, 4096, BIG}):
            if arena > 0 and arena != BIG:
                at[f"{t}:{arena}"] = run([t], arena)[0][0]
    bisected = []
    for k, t in enumerate(trials[:BISECTED]):
        lo, hi = 0, BIG                 # flagged at lo (0 bytes: any growth fails), clean at hi
        while hi - lo > 16:
            mid = (lo + hi) // 2 // 16 * 16
            if run([t], mid)[0][0][7] & ARENA_EXHAUSTED:
                lo = mid
            else:
                hi = mid
        bisected.append(hi)
    print(json.dumps({"big": big, "need": need, "at": at, "bisected": bisected, "slowest": slowest}))


if __name__ == "__main__":
    _worker(sys.argv[1], json.loads(sys.argv[2]))
    sys.exit(0)


# ------------------------------------------------------------------------------------------------ the tests
@pytest.fixture(scope="module")
def sanitized(tmp_path_factory):
    """tests/cmb_engine_host.cpp with ASan + UBSan (any report aborts the worker), and the environment that loads it"""
    so = tmp_path_factory.mktemp("arena") / "libcmb_engine_host_san.so"
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fno-omit-frame-pointer",
                    "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-shared", "-fPIC",
                    str(ROOT / "tests/cmb_engine_host.cpp"), "-o", str(so)], check=True, capture_output=True)
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], check=True, capture_output=True, text=True).stdout.strip()
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1:abort_on_error=1",
               UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    return str(so), env


def _run_worker(sanitized, job, timeout):
    so, env = sanitized
    p = subprocess.run([sys.executable, __file__, so, json.dumps(job)], env=env, capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0 and "Sanitizer" not in p.stderr and "runtime error" not in p.stderr, p.stderr[-4000:]
    out = json.loads(p.stdout.strip().splitlines()[-1])
    assert out["slowest"] < CALL_SECONDS, out["slowest"]
    return out


@pytest.mark.parametrize("name", list(SHAPES))
def test_a_trial_is_flagged_exactly_when_the_arena_is_smaller_than_it_needs(sanitized, name):
    c = SHAPES[name]
    trials = list(range(len(c["trials"])))
    r = _run_worker(sanitized, {"kind": "edges", "case": c, "trials": trials, "master": GOLD["master"]}, timeout=900)
    print(f"{name}: need per trial {r['need']} bytes")
    assert r["bisected"] == r["need"][:BISECTED]
    for k, t in enumerate(trials):
        need, big = r["need"][k], r["big"][k]
        assert need > 0, (name, t, "the shape grows no container")
        assert big[7] == 0, (name, t, big[7])
        want = c["trials"][t]
        if want is not None:
            check_trial(want, big[0], big[1], float.fromhex(big[2]), float.fromhex(big[3]), big[6], None, None, f"{name} trial {t}")
        for key, row in r["at"].items():
            tt, arena = map(int, key.split(":"))
            if tt != t:
                continue
            if arena < need:
                assert row[7] & ARENA_EXHAUSTED, (name, t, arena, need, row[7])
            else:
                assert row == big, (name, t, arena, need)


def _route_arena(cb, name):
    """The growth arena the shape's default route asks for: its workspace less the rings in front and the cursor's header"""
    import ctypes
    from cimba_b200 import _lib
    lib_model, _, variant, servers, _ = GPU_SHAPES[name]
    _, _, trials, nobj, _, _ = shape_of(name)
    if isinstance(lib_model, str):      # a model library built from examples/: the same formulas as the built-in routes
        lib_model = cb.MODEL_MM1
        variant = cb.VARIANT_STATIC if name.endswith("static") else cb.VARIANT_GENERAL
    job = _lib.DeviceJob(model=lib_model, servers=servers, variant=variant, num_trials=trials, num_objects=nobj)
    return int(_lib.lib.cimba_b200_workspace_bytes(ctypes.byref(job))) - rings_bytes(name, trials) - 256


@pytest.mark.parametrize("key", list(SAMPLED_NEED))
def test_the_gpu_shapes_need_at_least_twice_the_arena_their_routes_ask_for(sanitized, cb, key):
    names = [n for n in GPU_SHAPES if need_key(n) == key]
    host_model, servers, trials, nobj, arr, srv = shape_of(names[0])
    c = _case(host_model, servers, nobj, arr, srv)
    r = _run_worker(sanitized, {"kind": "need", "case": c, "trials": sample_trials(trials), "master": MASTER}, timeout=1800)
    need = r["need"]
    assert not any(r["status"])
    print(f"{key}: {trials} trials, sampled need per trial {min(need)}..{max(need)} bytes, sum of {SAMPLE} = {sum(need)}")
    assert sum(need) == SAMPLED_NEED[key]
    for name in names:
        arena = _route_arena(cb, name)
        print(f"  {name}: route arena {arena} bytes, estimated need {estimated_need(name)} ({estimated_need(name) / arena:.1f}x)")
        assert estimated_need(name) >= 2 * arena, (name, estimated_need(name), arena)
