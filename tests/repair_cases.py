"""Shared by tests/test_static_resources.py (CPU), tests/test_gpu_static_resources.py (GPU) and
tests/golden/make_repair_golden.py: the machine shop's stored vectors (tests/golden/repair_vectors.json) and its oracle,
oracle/_ref/librepairdrv.so - the same shop written against the unmodified reference (oracle/ref_build/repair_driver.c,
built by oracle/repair.mk).  params = [machines, exit while holding], as examples/repair_model.cuh reads them."""
import ctypes as C
import json
from pathlib import Path

from oracle_libs import Result

ROOT = Path(__file__).resolve().parents[1]
GOLD_PATH = ROOT / "tests/golden/repair_vectors.json"
GOLD = json.loads(GOLD_PATH.read_text()) if GOLD_PATH.exists() else None


def load_repair_ref():
    """oracle/_ref/librepairdrv.so, or None where it was not built (the reference sources are absent)."""
    so = ROOT / "oracle/_ref/librepairdrv.so"
    if not so.exists():
        return None
    lib = C.CDLL(str(so))
    lib.repair_ref_run_trials.restype = C.c_int
    lib.repair_ref_run_trials.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double,
                                          C.c_uint, C.c_int, C.POINTER(Result)]
    lib.repair_ref_trace_trial.restype = C.c_int
    lib.repair_ref_trace_trial.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_double, C.c_double, C.c_uint, C.c_int,
                                           C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double), C.POINTER(Result)]
    return lib


def machines(params):
    return int(params[0]) if len(params) > 0 and params[0] > 0 else 8


def ref_run(lib, servers, master, first, count, nobj, arr, srv, params):
    """Trials [first, first + count), seeds cmb_random_fmix64(master, global index)."""
    out = (Result * count)()
    rc = lib.repair_ref_run_trials(servers, master, first, count, nobj, arr, srv, machines(params),
                                   int(len(params) > 1 and params[1] != 0), out)
    assert rc == 0
    return list(out)


def ref_trace(lib, servers, seed, nobj, arr, srv, params, cap):
    """(result, keys, times) of one trial and its first `cap` pops."""
    r = Result()
    keys = (C.c_uint64 * max(cap, 1))()
    times = (C.c_double * max(cap, 1))()
    rc = lib.repair_ref_trace_trial(servers, seed, nobj, arr, srv, machines(params), int(len(params) > 1 and params[1] != 0),
                                    cap, keys, times, C.byref(r))
    assert rc == 0
    n = min(cap, r.events)
    return r, list(keys)[:n], list(times)[:n]
