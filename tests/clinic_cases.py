"""Shared by tests/test_model_random.py (CPU), tests/test_gpu_clinic.py (GPU) and tests/golden/make_clinic_golden.py: the
clinic's stored vectors (tests/golden/clinic_vectors.json) and its oracle, oracle/_ref/libclinicdrv.so - the clinic of
examples/clinic_model.cuh written against the unmodified reference (oracle/ref_build/clinic_driver.c, built by oracle/clinic.mk).
`report` (params[0]) picks the summary a trial writes to its counters: 0 queue, 1 signed values, 2 log / pow values, 3 group
sizes, 4 visit codes."""
import ctypes as C
import json
from pathlib import Path

from oracle_libs import Result

ROOT = Path(__file__).resolve().parents[1]
GOLD_PATH = ROOT / "tests/golden/clinic_vectors.json"
GOLD = json.loads(GOLD_PATH.read_text()) if GOLD_PATH.exists() else None
REPORTS = ("queue", "signed", "logpow", "sizes", "codes")
LOGPOW_REPORTS = (1, 2)             # summaries holding logistic, weibull, pareto and gamma-below-1 values: CUDA's log / pow


def load_clinic_ref():
    """oracle/_ref/libclinicdrv.so, or None where it was not built (the reference sources are absent)."""
    so = ROOT / "oracle/_ref/libclinicdrv.so"
    if not so.exists():
        return None
    lib = C.CDLL(str(so))
    lib.clinic_ref_run_trials.restype = C.c_int
    lib.clinic_ref_run_trials.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double, C.c_uint,
                                          C.POINTER(Result)]
    lib.clinic_ref_trace_trial.restype = C.c_int
    lib.clinic_ref_trace_trial.argtypes = [C.c_uint64, C.c_uint64, C.c_double, C.c_double, C.c_uint, C.c_uint64,
                                           C.POINTER(C.c_uint64), C.POINTER(C.c_double), C.POINTER(Result)]
    return lib


def ref_run(lib, master, first, count, nobj, arr, srv, report):
    """Trials [first, first + count), seeds cmb_random_fmix64(master, global index)."""
    out = (Result * count)()
    assert lib.clinic_ref_run_trials(master, first, count, nobj, arr, srv, report, out) == 0
    return list(out)


def ref_trace(lib, seed, nobj, arr, srv, report, cap):
    """(result, keys, times) of one trial and its first `cap` pops."""
    r = Result()
    keys = (C.c_uint64 * max(cap, 1))()
    times = (C.c_double * max(cap, 1))()
    assert lib.clinic_ref_trace_trial(seed, nobj, arr, srv, report, cap, keys, times, C.byref(r)) == 0
    k = min(r.events, cap)
    return r, list(keys[:k]), list(times[:k])
