"""GPU tests of the event list used as a whole (cmb_event_queue_initialize / _is_empty / _count / _clear, cmb_event_time /
_priority, cmb_event_pattern_find / _count / _cancel with the CMB_ANY_* wildcards): examples/event_model.cuh's two models, each
built for the general engine and for the static tier with scripts/build_model.py and loaded with cimba_b200_model_load -
EventTestT (the reference's own test/test_event.c) as examples/event_user_model.cu and examples/event_static_user_model.cu,
EventChurnT as examples/event_churn_user_model.cu and examples/event_churn_static_user_model.cu.

4096 trials of each model on each library, pop traces on: every trial identical row for row and trace for trace between the two
libraries; EventTestT's first 64 trials equal tests/golden/event_vectors.json (the unmodified reference); both models' first 64
equal the CPU build of the same source text (tests/event_queue_host.cpp).  diag[2] (trials the static library handed to the
general engine): every EventTestT trial (its wildcard loop finds three events at once), no EventChurnT trial."""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from event_cases import MASTER, TRACE_CAP, vectors
from test_event_queue import CHURN_MODEL, GENERAL, TEST_MODEL, HostResult, run

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
N = 4096
CHURN_OBJECTS, CHURN_SRV, CHURN_CAP = 40, 0.8, 1024       # EventChurnT: end at t = 40, holds of mean 0.8; fewer than 1024 pops


def _library(stem):
    so = ROOT / "cimba_b200/lib/models" / f"lib{stem}.so"
    if not so.exists():
        sys.path.insert(0, str(ROOT / "scripts"))
        import build_model
        build_model.build(ROOT / "examples" / f"{stem}.cu")
    return so


@pytest.fixture(scope="module")
def libs():
    ids = {name: cb.load_model(_library(stem)) for name, stem in (
        ("test_general", "event_user_model"), ("test_static", "event_static_user_model"),
        ("churn_general", "event_churn_user_model"), ("churn_static", "event_churn_static_user_model"))}
    assert cb.lib.cimba_b200_model_name(ids["test_static"]) == b"event"
    assert cb.lib.cimba_b200_model_name(ids["churn_static"]) == b"event_churn"
    return ids


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = tmp_path_factory.mktemp("event_queue_gpu") / "libevent_queue_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", str(ROOT / "tests/event_queue_host.cpp"),
                    "-o", str(so)], check=True, capture_output=True)
    lib = C.CDLL(str(so))
    lib.host_event_run_trials.restype = C.c_int
    lib.host_event_run_trials.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double,
                                          C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double), C.POINTER(HostResult)]
    return lib


def launch(model_id, cap, nobj=0, srv=1.0):
    """[(status, events, objects, t_end hex, counters, trace)] of trials 0..N-1, and diag[2]."""
    dev = torch.device("cuda", torch.cuda.current_device())
    arr = torch.ones(N, dtype=torch.float64, device=dev)
    srv = torch.full((N,), srv, dtype=torch.float64, device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(arr, srv, num_objects=nobj, master_seed=MASTER, model=model_id, trace_cap=cap, diag=diag)
    torch.cuda.synchronize()
    st = res.status.cpu().numpy()
    ev = res.events.cpu().numpy().astype(np.uint64)
    ob = res.objects.cpu().numpy().astype(np.uint64)
    te = res.t_end.cpu().numpy()
    co = res.counters.cpu().numpy().astype(np.uint64)
    tk = res.trace_key.cpu().numpy().astype(np.uint64).reshape(N, cap)
    tt = res.trace_time.cpu().numpy().reshape(N, cap)
    rows = []
    for i in range(N):
        n = min(int(ev[i]), cap)
        rows.append((int(st[i]), int(ev[i]), int(ob[i]), float(te[i]).hex(), [int(v) for v in co[i]],
                     [(int(k), float(t).hex()) for k, t in zip(tk[i, :n], tt[i, :n])]))
    return rows, int(diag[2].item())


def test_event_test_on_both_libraries(libs, host):
    general, handed_g = launch(libs["test_general"], TRACE_CAP)
    static, handed_s = launch(libs["test_static"], TRACE_CAP)
    print(f"EventTestT: diag[2] general {handed_g}, static {handed_s} of {N}")
    assert handed_g == 0 and handed_s == N
    assert all(r[0] == 0 and r[1] < TRACE_CAP for r in general)
    assert static == general
    want = vectors()["trials"]
    for i, w in enumerate(want):
        g = general[i]
        assert (g[1], g[3], g[4]) == (w["events"], w["t_end"], w["counters"]), i
        assert g[5] == [tuple(x) for x in w["trace"]], i
    assert general[:64] == run(host, TEST_MODEL, GENERAL, 64, cap=TRACE_CAP)


def test_event_churn_on_both_libraries(libs, host):
    general, handed_g = launch(libs["churn_general"], CHURN_CAP, CHURN_OBJECTS, CHURN_SRV)
    static, handed_s = launch(libs["churn_static"], CHURN_CAP, CHURN_OBJECTS, CHURN_SRV)
    print(f"EventChurnT: diag[2] general {handed_g}, static {handed_s} of {N}")
    assert handed_g == 0 and handed_s == 0
    assert all(r[0] == 0 and r[1] < CHURN_CAP for r in general)
    assert static == general
    assert len({r[1] for r in general[:32]}) > 8                   # the trials of a warp differ
    assert general[:64] == run(host, CHURN_MODEL, GENERAL, 64, num_objects=CHURN_OBJECTS, srv_mean=CHURN_SRV, cap=CHURN_CAP)
