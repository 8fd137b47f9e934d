"""cimba_b200_launch, job by job: which route serves a job shows in its return code, the refusal text and how many kernels it
starts (cimba_b200_launch_count, which bench.py reports as gpu_launches).  Every model id 0-22 with variants 0-4, 16 and 17
(0 and 16 where the variant picks nothing), with and without a status array, then one job for each refusal a route makes (mapping, servers out of range, workspace one
byte short, MM1_RECORDED without counters, AWACS without a duration, an invalid spill cap, unknown ids) and a few traced and
warp-mapped launches.  Every refused job is refused on the host, before any kernel starts.

The expected table was recorded on an H100 from the library as it was before its routes were gathered into one table
(record_launch_table below)."""
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from cimba_b200 import _lib

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
FIXTURE = ROOT / "tests" / "golden" / "launch_routes_launches.json"
TRIALS, TRACE_CAP = 8, 16
GEN, STA = cb.VARIANT_GENERAL, cb.VARIANT_STATIC
VARIANTS = (0, 1, 2, 3, 4, GEN, STA)
# model -> (servers, num_objects, params): short trials; num_objects is the duration of the time-bounded models
SHAPE = {0: (1, 200, ()), 1: (1, 200, ()), 2: (3, 200, ()), 3: (10, 50, ()), 4: (20, 50, ()), 5: (10, 50, ()), 6: (8, 50, ()),
         7: (64, 5, ()), 8: (1, 50, ()), 9: (1, 200, ()), 10: (6, 24, ()), 11: (10, 50, ()), 12: (10, 50, ()), 13: (10, 50, ()),
         14: (1, 50, ()), 15: (0, 60, ()), 16: (40, 50, (0.7,)), 17: (1, 200, ()), 18: (20, 100, ()), 19: (1, 500, (10.0,)),
         20: (1, 0, ()), 21: (1, 0, ()), 22: (1, 200, ())}
ROUTED_BY_VARIANT = (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 19)     # the others run one way whatever the variant
USER_LIB = "mm1_user_model"


def _cases():
    """name -> (model, variant, overrides).  Overrides: job fields, plus status=False, counters=False, trace=True,
    short=True (workspace one byte short)."""
    c = {}
    for m in SHAPE:
        if m == 21:                                     # tutorial 2's trials have a fixed length: about 30 s per launch
            c["m21_v0"] = (m, 0, {})
            continue
        for v in (VARIANTS if m in ROUTED_BY_VARIANT else (0, GEN)):
            c[f"m{m}_v{v}"] = (m, v, {})
            c[f"m{m}_v{v}_nostatus"] = (m, v, {"status": False})
    warp = {"mapping": cb.MAP_WARP}
    for m, v in ((0, 0), (1, 0), (9, 0), (0, 1), (1, 1), (0, 2), (0, GEN), (0, STA), (19, 0), (2, 0), (2, GEN), (3, 0), (3, GEN),
                 (8, 0), (10, 0), (10, GEN), (16, 0), (7, 0), (15, 0)):
        c[f"m{m}_v{v}_warp"] = (m, v, warp)
    for m, v, s in ((2, 0, 0), (2, 0, 15), (2, 1, 15), (3, 0, 0), (3, 0, 17), (3, GEN, 0), (6, 0, 16), (13, 0, 16), (11, 0, 17),
                    (4, 0, 0), (4, 0, 100), (8, 0, 0), (8, GEN, 0), (14, GEN, 0), (16, 0, 0), (0, GEN, 0), (10, 0, 2), (10, 0, 256),
                    (10, 2, 255), (10, GEN, 0), (10, GEN, 2), (7, 0, 0), (7, 1, 1081), (7, 1, 1080), (7, 0, 33822), (7, 0, 33823),
                    (7, 3, 40000)):
        c[f"m{m}_v{v}_servers{s}"] = (m, v, {"servers": s})
    for m, v in ((0, 0), (0, 1), (0, 2), (0, GEN), (0, STA), (1, 0), (9, 0), (2, 0), (2, GEN), (3, 0), (3, GEN), (8, 0), (10, 0),
                 (10, 1), (10, GEN), (15, 0), (7, 0), (7, 2), (19, 0), (19, GEN), (16, 0), (18, 0), (20, 0), (21, 0)):
        c[f"m{m}_v{v}_short"] = (m, v, {"short": True})
    for v in (0, 1, 2, GEN, STA):
        c[f"m9_v{v}_nocounters"] = (9, v, {"counters": False})
    c["m15_v0_duration0"] = (15, 0, {"num_objects": 0})
    for m, v in ((0, 0), (0, STA), (2, 0), (3, 0), (10, 0)):
        c[f"m{m}_v{v}_spill3"] = (m, v, {"queue_spill_cap": 3})
        c[f"m{m}_v{v}_spill8192"] = (m, v, {"queue_spill_cap": 8192})
    for m, v in ((0, 0), (0, 1), (0, 2), (0, STA), (1, 0), (9, 0), (2, 0), (2, 1), (3, 0), (8, 0), (10, 0), (10, 1), (10, GEN),
                 (7, 0), (7, 1), (7, 2), (7, 3), (7, 4), (19, 0), (16, 0), (15, 0)):
        c[f"m{m}_v{v}_trace"] = (m, v, {"trace": True})
    for m in (-1, 1000 + 4095):
        c[f"m{m}_unknown"] = (m, 0, {})
    for name, o in (("", {}), ("_nostatus", {"status": False}), ("_short", {"short": True}), ("_warp", warp)):
        c[f"user{name}"] = ("user", 0, o)
    return c


CASES = _cases()


def _setup():
    torch.cuda.set_device(0)
    # a flat terrain of the library's own (MODEL_AWACS reads the one registered for the device)
    cb.awacs_upload_terrain(np.zeros(64 * 64, dtype=np.float32), 64, 64, (30.0, 30.0, -1e6, 1e6, -1e6, 1e6))
    return {"user": cb.load_model(ROOT / "cimba_b200/lib/models" / f"lib{USER_LIB}.so")}


@pytest.fixture(scope="module")
def ready():
    return _setup()


def _run(case, ids):
    """(return code, cimba_b200_last_error text or None, kernels started) of one job, after the device finished it."""
    model, variant, o = CASES[case]
    servers, nobj, params = SHAPE.get(0 if model == "user" else model, (1, 200, ()))
    dev = torch.device("cuda", 0)
    f64 = lambda: torch.zeros(TRIALS, dtype=torch.float64, device=dev)
    u64 = lambda k=1: torch.zeros(TRIALS * k, dtype=torch.int64, device=dev)
    u32 = lambda: torch.zeros(TRIALS, dtype=torch.int32, device=dev)
    arr, srv = torch.full((TRIALS,), 1.25, dtype=torch.float64, device=dev), torch.full((TRIALS,), 1.0, dtype=torch.float64, device=dev)
    keep = [arr, srv, f64(), f64(), u64(), u64(), u32(), u32(), u64(8), u64(TRACE_CAP), f64()]
    pars = (C.c_double * max(1, len(params)))(*params)
    job = _lib.DeviceJob(model=ids["user"] if model == "user" else model, servers=o.get("servers", servers), variant=variant,
                         mapping=o.get("mapping", 0), master_seed=0x5DEECE66D2B3F10B, first_trial=3, num_trials=TRIALS,
                         num_objects=o.get("num_objects", nobj), arr_mean=arr.data_ptr(), srv_mean=srv.data_ptr(),
                         t_end=keep[2].data_ptr(), sum_wait=keep[3].data_ptr(), events=keep[4].data_ptr(), objects=keep[5].data_ptr(),
                         status=keep[6].data_ptr() if o.get("status", True) else None, max_queue=keep[7].data_ptr(),
                         counters=keep[8].data_ptr() if o.get("counters", True) else None,
                         queue_spill_cap=o.get("queue_spill_cap", 0), params=pars, num_params=len(params))
    if o.get("trace"):
        keep += [u64(TRACE_CAP), f64().repeat(TRACE_CAP)]
        job.trace_cap, job.trace_key, job.trace_time = TRACE_CAP, keep[-2].data_ptr(), keep[-1].data_ptr()
    need = int(_lib.lib.cimba_b200_workspace_bytes(C.byref(job)))
    ws = torch.empty(max(need, 256), dtype=torch.uint8, device=dev)
    job.workspace, job.workspace_bytes = ws.data_ptr(), need - 1 if o.get("short") else need
    before = int(_lib.lib.cimba_b200_launch_count())
    rc = int(_lib.lib.cimba_b200_launch(C.byref(job), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    launches = int(_lib.lib.cimba_b200_launch_count()) - before
    torch.cuda.synchronize(dev)
    return {"rc": rc, "err": _lib.lib.cimba_b200_last_error().decode() if rc != 0 else None, "launches": launches}


def record_launch_table():
    """Rewrite the fixture on a GPU: PYTHONPATH=. CIMBA_B200_LIB=path/to/libcimba_b200.so python tests/test_gpu_launch_routes.py --record"""
    import time
    ids, table = _setup(), {}
    for k in CASES:
        t0 = time.perf_counter()
        table[k] = _run(k, ids)
        print(k, table[k], f"{time.perf_counter() - t0:.2f} s", flush=True)
    FIXTURE.write_text(json.dumps(table, indent=0, sort_keys=True) + "\n")


@pytest.fixture(scope="module")
def want():
    table = json.loads(FIXTURE.read_text())
    assert sorted(table) == sorted(CASES)
    return table


GROUPS = sorted({k.split("_")[0] for k in CASES})


@pytest.mark.parametrize("group", GROUPS)
def test_launch_routes_as_recorded(ready, want, group):
    names = [k for k in CASES if k.split("_")[0] == group]
    got = {k: _run(k, ready) for k in names}
    bad = {k: (want[k], got[k]) for k in names if got[k] != want[k]}
    assert not bad, bad
    for k in names:                                     # a refusal starts nothing
        assert got[k]["rc"] == 0 or got[k]["launches"] == 0, k


if __name__ == "__main__":
    if sys.argv[1:] != ["--record"]:
        sys.exit(record_launch_table.__doc__)
    record_launch_table()
