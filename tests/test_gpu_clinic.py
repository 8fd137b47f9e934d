"""GPU tests of examples/clinic_model.cuh - a walk-in clinic that draws every cmb_random distribution model code has, triages by
a Vose alias table and keeps cmb_datasummary / cmb_wtdsummary statistics - built twice with scripts/build_model.py and loaded
with cimba_b200_model_load: on the general engine (examples/clinic_user_model.cu) and on the static tier
(examples/clinic_static_user_model.cu, cmb::StaticSim<4, 2>, whose sampled holds are drawn rectangles first).

Both libraries must reproduce the vectors of the same clinic written against the unmodified reference
(tests/golden/clinic_vectors.json, oracle/ref_build/clinic_driver.c), pop traces included, and agree with each other bit for bit
on 3072 trials with drawn means - and with the model's source text run on the CPU (tests/model_random_host.cpp) and the live
reference build where it travelled.  The summaries of logistic, weibull, pareto and gamma-below-1 values (reports 1 and 2) hold
CUDA's log / pow where the reference has glibc's: they agree to within rounding (relative 1e-12).
cimba_b200_merge_weighted_rows over the per-trial rows equals the same merge tree on the host.  diag[2] (trials the static
library handed to the general engine) is reported."""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from clinic_cases import GOLD, LOGPOW_REPORTS, REPORTS, load_clinic_ref, ref_run
from cmb_cases import trace_digest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
MASTER = GOLD["master"]
NOBJ, ARR, SRV = 300, 2.0, 0.6
CASES = {c["name"]: c for c in GOLD["cases"]}


def _library(stem):
    so = ROOT / "cimba_b200/lib/models" / f"lib{stem}.so"
    if not so.exists():
        sys.path.insert(0, str(ROOT / "scripts"))
        import build_model
        build_model.build(ROOT / "examples" / f"{stem}.cu")
    return so


@pytest.fixture(scope="module")
def libs():
    static = cb.load_model(_library("clinic_static_user_model"))
    general = cb.load_model(_library("clinic_user_model"))
    assert cb.lib.cimba_b200_model_name(static) == b"clinic"
    return {"static": static, "general": general}


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    sys.path.insert(0, str(ROOT / "tests"))
    from test_model_random import HostResult
    so = tmp_path_factory.mktemp("clinic") / "libmodel_random_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", str(ROOT / "tests/model_random_host.cpp"),
                    "-o", str(so)], check=True, capture_output=True)
    lib = C.CDLL(str(so))
    lib.host_clinic_run_trials.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double,
                                           C.c_double, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double),
                                           C.POINTER(HostResult)]
    return lib, HostResult


def launch(model_id, n, report, first=0, nobj=NOBJ, arr=ARR, srv=SRV, trace=0):
    dev = torch.device("cuda", torch.cuda.current_device())
    arr = torch.as_tensor(np.broadcast_to(np.asarray(arr, dtype=np.float64), (n,)).copy(), device=dev)
    srv = torch.as_tensor(np.broadcast_to(np.asarray(srv, dtype=np.float64), (n,)).copy(), device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(arr, srv, num_objects=nobj, master_seed=MASTER, first_trial=first, model=model_id,
                           queue_spill_cap=4096, trace_cap=trace, params=[report], diag=diag)
    torch.cuda.synchronize()
    return res, int(diag[2].item())


def rows(res):
    return [(int(s), int(e), int(o), float(t).hex(), float(w).hex(), [int(v) for v in c])
            for s, e, o, t, w, c in zip(res.status.cpu().numpy(), res.events.cpu().numpy().astype(np.uint64),
                                        res.objects.cpu().numpy().astype(np.uint64), res.t_end.cpu().numpy(),
                                        res.sum_wait.cpu().numpy(), res.counters.cpu().numpy().astype(np.uint64))]


def _f(u):
    return np.array([u], dtype=np.uint64).view(np.float64)[0]


def same_row(got, want, report, what):
    if report in LOGPOW_REPORTS:
        assert got[0] == want[0], what
        np.testing.assert_allclose([_f(v) for v in got[1:]], [_f(v) for v in want[1:]], rtol=1e-12, atol=0.0, err_msg=str(what))
    else:
        assert got == want, what


@pytest.mark.parametrize("report", range(len(REPORTS)), ids=REPORTS)
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("engine", ["static", "general"])
def test_clinic_on_device_matches_the_reference_vectors(libs, engine, name, report):
    """Every vector trial: events, patients served, clock, time in clinic, the pop trace and the eight counters of summary
    `report`; status 0, and no trial handed on by the static library."""
    case = CASES[name]
    n = len(case["trials"])
    res, handed = launch(libs[engine], n, report, nobj=case["num_objects"], arr=float.fromhex(case["arr_mean"]),
                         srv=float.fromhex(case["srv_mean"]), trace=GOLD["trace"])
    assert handed == 0, (engine, name, handed)
    tk, tt = res.trace_key.cpu().numpy(), res.trace_time.cpu().numpy()
    for i, (got, want) in enumerate(zip(rows(res), case["trials"])):
        what = (engine, name, report, i)
        assert got[:5] == (0, want["events"], want["objects"], want["t_end"], want["sum_wait"]), what
        assert trace_digest(tk[i], tt[i], got[1]) == want["trace_sha256"], (what, "pop trace")
        same_row(got[5], want["rows"][report], report, what)


@pytest.fixture(scope="module")
def drawn():
    """3072 trials from first_trial 911, each with its own drawn means (every warp mixes loads)."""
    rnd = np.random.default_rng(20261017)
    n = 3072
    return n, 911, rnd.choice([1.2, 1.6, 2.0, 3.0, 3.5], n), rnd.choice([0.3, 0.45, 0.6, 0.9], n)


@pytest.mark.parametrize("report", range(len(REPORTS)), ids=REPORTS)
def test_drawn_trials_static_equals_general_equals_host_and_reference(libs, host, drawn, report):
    """The drawn trials: static library = general library bit for bit; the first 96 = the CPU build of the model text and the
    live reference build where it travelled (rows of reports 1 and 2 to within rounding)."""
    n, first, arr, srv = drawn
    got = {}
    for engine in ("static", "general"):
        res, handed = launch(libs[engine], n, report, first, arr=arr, srv=srv)
        got[engine] = rows(res)
        print(f"report {report}: {engine} library, diag[2] (trials handed to the general engine) = {handed}")
        assert handed == 0
    assert got["static"] == got["general"]
    assert all(r[0] == 0 for r in got["static"])
    assert len({r[1] for r in got["static"][:32]}) > 16             # the trials of a warp differ
    lib, HostResult = host
    ref = load_clinic_ref()
    for i in range(96):
        out = (HostResult * 1)()
        assert lib.host_clinic_run_trials(1, MASTER, first + i, 1, NOBJ, float(arr[i]), float(srv[i]), float(report), 0, 0,
                                          None, None, out) == 0
        o = out[0]
        g = got["static"][i]
        assert g[:5] == (o.status, o.events, o.objects, o.t_end.hex(), o.sum_wait.hex()), (report, i)
        same_row(g[5], list(o.counter), report, (report, i, "host"))
        if ref is not None:
            w = ref_run(ref, MASTER, first + i, 1, NOBJ, float(arr[i]), float(srv[i]), report)[0]
            assert g[:5] == (0, w.events, w.objects, w.t_end.hex(), w.sum_wait.hex()), (report, i, "reference")
            same_row(g[5], list(w.counter), report, (report, i, "reference"))


def test_merge_weighted_rows_equals_the_host_merge(libs):
    """cimba_b200_merge_weighted_rows over 1000 trials' rows (summary 0, the queue history) equals the same fixed tree of
    cimba_b200_wtdsummary_merge on the host: thread t folds rows t, t + 256, ...; then halving merges."""
    res, _ = launch(libs["static"], 1000, 0)
    dev_row = cb.merge_weighted_rows_on_device(res.counters).cpu().numpy().astype(np.uint64).tolist()
    from cimba_b200 import _lib
    raw = C.CDLL(str(_lib.LIB_PATH))
    WS = _lib.WtdSummaryStruct
    cnt = res.counters.cpu().numpy().astype(np.uint64)

    def load(r):
        s = WS()
        raw.cimba_b200_wtdsummary_initialize(C.byref(s))
        s.base.count = int(r[0])
        s.base.min, s.base.max, s.base.m1, s.base.m2, s.base.m3, s.base.m4, s.wsum = (_f(v) for v in r[1:])
        return s

    part = []
    for t in range(256):
        acc = WS()
        raw.cimba_b200_wtdsummary_initialize(C.byref(acc))
        for i in range(t, len(cnt), 256):
            nxt = WS()
            raw.cimba_b200_wtdsummary_merge(C.byref(nxt), C.byref(acc), C.byref(load(cnt[i])))
            acc = nxt
        part.append(acc)
    s = 128
    while s > 0:
        for t in range(s):
            nxt = WS()
            raw.cimba_b200_wtdsummary_merge(C.byref(nxt), C.byref(part[t]), C.byref(part[t + s]))
            part[t] = nxt
        s //= 2
    c = part[0]
    bits = [int(np.array([v], dtype=np.float64).view(np.uint64)[0])
            for v in (c.base.min, c.base.max, c.base.m1, c.base.m2, c.base.m3, c.base.m4, c.wsum)]
    assert dev_row == [c.base.count] + bits


def test_host_buffer_entry_equals_the_device_entry(libs):
    """cimba_run_experiment over a host array with a counters field: the same trials as launch_trials, on both libraries."""
    dt = np.dtype([("arr_mean", "<f8"), ("srv_mean", "<f8"), ("obj_cnt", "<u8"), ("sum_wait", "<f8"), ("events", "<u8"),
                   ("t_end", "<f8"), ("status", "<u4"), ("pad", "<u4"), ("counters", "<u8", (8,))])
    for engine in ("static", "general"):
        dev, _ = launch(libs[engine], 200, 3, first=5)
        exp = np.zeros(200, dtype=dt)
        exp["arr_mean"], exp["srv_mean"] = ARR, SRV
        cb.cimba_run_experiment(exp, model=libs[engine], num_objects=NOBJ, master_seed=MASTER, first_trial=5,
                                queue_spill_cap=4096, params=[3])
        assert not exp["status"].any()
        host = [(0, int(e["events"]), int(e["obj_cnt"]), float(e["t_end"]).hex(), float(e["sum_wait"]).hex(),
                 [int(v) for v in e["counters"]]) for e in exp]
        assert host == rows(dev), engine
