"""ctypes binding of the C-ABI library declared in include/cimba_b200.h.

The shared object is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).
There is no Python or CPU implementation behind these calls: if the library is
missing, importing this module raises.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import os

# CIMBA_B200_LIB selects an alternative build of the same library (tuning sweeps)
LIB_PATH = Path(os.environ.get("CIMBA_B200_LIB") or
                Path(__file__).resolve().parent / "lib" / "libcimba_b200.so")

NO_FIELD = C.c_size_t(-1).value

MODEL_MM1, MODEL_GG1, MODEL_MMC, MODEL_GUARDED, MODEL_PREEMPT, MODEL_BUFFER, MODEL_PRIOQ, MODEL_HOLD, MODEL_TIMERS, MODEL_MM1_RECORDED, MODEL_HARBOR, MODEL_GUARDED_RECORDED, MODEL_BUFFER_RECORDED, MODEL_PRIOQ_RECORDED, MODEL_RESOURCE_RECORDED, MODEL_AWACS = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15
MODEL_RENEGE, MODEL_POOL_RECORDED, MODEL_TUTORIAL1, MODEL_PARK, MODEL_TUTORIAL2, MODEL_USER_BASE, VARIANT_GENERAL, VARIANT_STATIC = 16, 18, 19, 20, 21, 1000, 16, 17
MAP_LANE, MAP_WARP = 1, 32

OK, EINVAL, ENODEVICE, ECUDA, ETRIAL, ENOMEM = 0, -1, -2, -3, -4, -5

# a trial's status word: CIMBA_B200_TRIAL_* bits
(TRIAL_QUEUE_OVERFLOW, TRIAL_FEL_OVERFLOW, TRIAL_KEY_OVERFLOW, TRIAL_GUARD_OVERFLOW, TRIAL_PROC_OVERFLOW, TRIAL_NEGATIVE_HOLD,
 TRIAL_ARENA_EXHAUSTED, TRIAL_BAD_ARGUMENT) = 1, 2, 4, 8, 16, 32, 64, 128


class DeviceJob(C.Structure):
    """struct cimba_b200_device_job"""
    _fields_ = [
        ("model", C.c_int32), ("servers", C.c_int32), ("mapping", C.c_int32), ("variant", C.c_int32),
        ("master_seed", C.c_uint64), ("first_trial", C.c_uint64),
        ("num_trials", C.c_uint64), ("num_objects", C.c_uint64),
        ("arr_mean", C.c_void_p), ("srv_mean", C.c_void_p),
        ("events", C.c_void_p), ("objects", C.c_void_p),
        ("t_end", C.c_void_p), ("sum_wait", C.c_void_p),
        ("status", C.c_void_p), ("max_queue", C.c_void_p), ("counters", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_uint64),
        ("trace_cap", C.c_uint64), ("trace_key", C.c_void_p), ("trace_time", C.c_void_p),
        ("queue_spill_cap", C.c_uint32), ("reserved0", C.c_uint32), ("diag", C.c_void_p),
        ("params", C.POINTER(C.c_double)), ("num_params", C.c_uint32), ("reserved1", C.c_uint32),
    ]


class AwacsTerrain(C.Structure):
    """struct cimba_b200_awacs_terrain"""
    _fields_ = [("map", C.c_void_p), ("cols", C.c_uint32), ("rows", C.c_uint32),
                ("x_scale", C.c_float), ("y_scale", C.c_float),
                ("x_min", C.c_float), ("x_max", C.c_float), ("y_min", C.c_float), ("y_max", C.c_float)]


THREAD_INIT_FUNC = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_uint64)     # cimba_thread_init_func, include/cimba.h:155
THREAD_EXIT_FUNC = C.CFUNCTYPE(None, C.c_void_p)                      # cimba_thread_exit_func, :163


class Experiment(C.Structure):
    """struct cimba_b200_experiment"""
    _fields_ = [
        ("model", C.c_int32), ("servers", C.c_int32), ("mapping", C.c_int32), ("device", C.c_int32),
        ("variant", C.c_int32), ("queue_spill_cap", C.c_uint32),
        ("master_seed", C.c_uint64), ("first_trial", C.c_uint64), ("num_objects", C.c_uint64),
        ("off_arr_mean", C.c_size_t), ("off_srv_mean", C.c_size_t),
        ("off_obj_cnt", C.c_size_t), ("off_sum_wait", C.c_size_t), ("off_avg_wait", C.c_size_t),
        ("off_events", C.c_size_t), ("off_t_end", C.c_size_t), ("off_status", C.c_size_t),
        ("off_max_queue", C.c_size_t), ("off_counters", C.c_size_t),
        ("params", C.POINTER(C.c_double)), ("num_params", C.c_uint32), ("reserved", C.c_uint32),
    ]


class DataSummaryStruct(C.Structure):
    """struct cimba_b200_datasummary == reference struct cmb_datasummary layout"""
    _fields_ = [
        ("cookie", C.c_uint64), ("count", C.c_uint64),
        ("min", C.c_double), ("max", C.c_double),
        ("m1", C.c_double), ("m2", C.c_double), ("m3", C.c_double), ("m4", C.c_double),
    ]


class WtdSummaryStruct(C.Structure):
    """struct cimba_b200_wtdsummary == reference struct cmb_wtdsummary layout"""
    _fields_ = [("base", DataSummaryStruct), ("wsum", C.c_double)]


# every symbol include/cimba_b200.h declares: (restype, argtypes)
SYMBOLS = {
    "cimba_b200_workspace_bytes": (C.c_uint64, [C.POINTER(DeviceJob)]),
    "cimba_b200_launch": (C.c_int, [C.POINTER(DeviceJob), C.c_void_p]),
    "cimba_b200_launch_count": (C.c_uint64, []),
    "cimba_b200_mm1_resident_ctas": (C.c_int, [C.c_int]),
    "cimba_b200_summarize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "cimba_b200_run_experiment": (C.c_int, [C.c_void_p, C.c_uint64, C.c_size_t, C.POINTER(Experiment)]),
    "cimba_b200_release_cache": (None, []),
    "cimba_b200_run_experiment_all_gpus": (C.c_int, [C.c_void_p, C.c_uint64, C.c_size_t, C.POINTER(Experiment),
                                                     C.c_int]),
    "cimba_b200_awacs_set_terrain": (C.c_int, [C.POINTER(AwacsTerrain)]),
    "cimba_b200_awacs_upload_terrain": (C.c_int, [C.POINTER(AwacsTerrain)]),
    "cimba_b200_set_thread_hooks": (None, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "cimba_b200_thread_context": (C.c_void_p, []),
    "cimba_b200_datasummary_initialize": (None, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_add": (C.c_uint64, [C.POINTER(DataSummaryStruct), C.c_double]),
    "cimba_b200_datasummary_merge": (C.c_uint64, [C.POINTER(DataSummaryStruct)] * 3),
    "cimba_b200_datasummary_mean": (C.c_double, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_variance": (C.c_double, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_stddev": (C.c_double, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_count": (C.c_uint64, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_max": (C.c_double, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_min": (C.c_double, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_skewness": (C.c_double, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_kurtosis": (C.c_double, [C.POINTER(DataSummaryStruct)]),
    "cimba_b200_datasummary_print": (None, [C.POINTER(DataSummaryStruct), C.c_void_p, C.c_int]),
    "cimba_b200_summarize_weighted": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "cimba_b200_merge_weighted_rows": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "cimba_b200_wtdsummary_initialize": (None, [C.POINTER(WtdSummaryStruct)]),
    "cimba_b200_wtdsummary_add": (C.c_uint64, [C.POINTER(WtdSummaryStruct), C.c_double, C.c_double]),
    "cimba_b200_wtdsummary_merge": (C.c_uint64, [C.POINTER(WtdSummaryStruct)] * 3),
    "cimba_b200_wtdsummary_mean": (C.c_double, [C.POINTER(WtdSummaryStruct)]),
    "cimba_b200_wtdsummary_variance": (C.c_double, [C.POINTER(WtdSummaryStruct)]),
    "cimba_b200_wtdsummary_stddev": (C.c_double, [C.POINTER(WtdSummaryStruct)]),
    "cimba_b200_wtdsummary_skewness": (C.c_double, [C.POINTER(WtdSummaryStruct)]),
    "cimba_b200_wtdsummary_kurtosis": (C.c_double, [C.POINTER(WtdSummaryStruct)]),
    "cimba_b200_wtdsummary_print": (None, [C.POINTER(WtdSummaryStruct), C.c_void_p, C.c_int]),
    "cimba_b200_fmix64": (C.c_uint64, [C.c_uint64, C.c_uint64]),
    "cimba_b200_rng_draws": (C.c_int, [C.c_uint64, C.c_int, C.c_double, C.c_double,
                                       C.c_uint64, C.c_void_p, C.c_void_p]),
    "cimba_b200_rng_draws_ex": (C.c_int, [C.c_uint64, C.c_int, C.POINTER(C.c_double), C.c_uint32,
                                          C.c_uint64, C.c_void_p, C.c_void_p]),
    "cimba_b200_alias_create": (C.c_int, [C.c_uint32, C.POINTER(C.c_double), C.POINTER(C.c_uint64),
                                          C.POINTER(C.c_uint32)]),
    "cimba_b200_model_load": (C.c_int, [C.c_char_p]),
    "cimba_b200_model_name": (C.c_char_p, [C.c_int]),
    "cimba_b200_version": (C.c_char_p, []),
    "cimba_b200_last_error": (C.c_char_p, []),
    "cimba_b200_device_count": (C.c_int, []),
}


# diagnostics that builds older than this binding lack (CIMBA_B200_LIB may select one to compare against): left unbound there
DIAGNOSTICS = {"cimba_b200_mm1_resident_ctas"}


def load() -> C.CDLL:
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). cimba_b200 has no CPU fallback.")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SYMBOLS.items():
        if name in DIAGNOSTICS and not hasattr(lib, name):
            continue
        fn = getattr(lib, name)          # AttributeError if the export is missing
        fn.restype = res
        fn.argtypes = args
    return lib


lib = load()


class CimbaError(RuntimeError):
    def __init__(self, code: int):
        self.code = code
        msg = lib.cimba_b200_last_error().decode(errors="replace")
        super().__init__(f"cimba_b200 error {code}: {msg}")


def check(code: int) -> None:
    if code != OK:
        raise CimbaError(code)
