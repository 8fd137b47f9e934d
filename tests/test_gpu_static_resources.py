"""GPU tests of cmb_resourcepool and cmb_resource on the static tier (cimba_b200/csrc/cmb_static.cuh).

examples/repair_model.cuh - machines sharing a repair crew (a pool, its usage history on) and an inspection bench (a resource)
- built twice with scripts/build_model.py and loaded with cimba_b200_model_load: on the general engine
(examples/repair_user_model.cu) and on the static tier (examples/repair_static_user_model.cu, cmb::StaticSim<8, 0>, whose
launch re-runs on the general engine whatever the tier flags).  Both must reproduce the unmodified reference bit for bit
(tests/golden/repair_vectors.json; the live build oracle/_ref/librepairdrv.so where it travelled), pop traces included.
diag[2] counts the trials the static library handed to the general engine: none where the shop fits the tier, all of them
with twelve machines and with machines that exit holding crew."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from cmb_cases import trace_digest
from repair_cases import GOLD, load_repair_ref, ref_run

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
MASTER, TRACE = GOLD["master"], GOLD["trace"]
FALLBACK = ("twelve_machines", "exit_holding")
CASES = {c["name"]: c for c in GOLD["cases"]}

# per-trial parameters in the manner of tests/param_cases.py: periods 7 and 5, so every warp mixes loads; srv_mean never 1.0
FIRST, N = 4093, 197
UP = (4.0, 2.5, 7.0, 3.1, 12.0, 1.7, 5.5)
REPAIR = (0.37, 1.3, 0.61, 0.93, 2.2)


def _library(stem):
    so = ROOT / "cimba_b200/lib/models" / f"lib{stem}.so"
    if not so.exists():                                 # built by __graft_entry__.build(); nvcc is on the GPU machine too
        sys.path.insert(0, str(ROOT / "scripts"))
        import build_model
        build_model.build(ROOT / "examples" / f"{stem}.cu")
    return so


@pytest.fixture(scope="module")
def libs():
    static = cb.load_model(_library("repair_static_user_model"))
    general = cb.load_model(_library("repair_user_model"))
    assert cb.lib.cimba_b200_model_name(static) == b"repair"
    return {"static": static, "general": general}


def launch(model_id, arr, srv, case, first=0, trace=TRACE):
    dev = torch.device("cuda", torch.cuda.current_device())
    arr = torch.as_tensor(np.asarray(arr, dtype=np.float64), device=dev)
    srv = torch.as_tensor(np.asarray(srv, dtype=np.float64), device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(arr, srv, num_objects=case["num_objects"], master_seed=MASTER, first_trial=first, model=model_id,
                           servers=case["servers"], trace_cap=trace, params=case["params"], diag=diag)
    torch.cuda.synchronize()
    return res, int(diag[2].item())


def rows(res):
    cnt = res.counters.cpu().numpy().astype(np.uint64)
    return [(int(e), int(o), float(t).hex(), float(s).hex(), [int(v) for v in c])
            for e, o, t, s, c in zip(res.events.cpu().numpy().astype(np.uint64), res.objects.cpu().numpy().astype(np.uint64),
                                     res.t_end.cpu().numpy(), res.sum_wait.cpu().numpy(), cnt)]


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("engine", ["static", "general"])
def test_repair_shop_on_device_matches_the_reference_vectors(libs, engine, name):
    case = CASES[name]
    n = len(case["trials"])
    res, repaired = launch(libs[engine], [float.fromhex(case["arr_mean"])] * n, [float.fromhex(case["srv_mean"])] * n, case)
    # the proof of which engine answered: the static library ran every in-tier trial itself, and handed on every other one
    assert repaired == (n if engine == "static" and name in FALLBACK else 0), (engine, name, repaired)
    assert (res.status.cpu().numpy() == 0).all(), res.status.cpu().numpy()
    tk, tt = res.trace_key.cpu().numpy(), res.trace_time.cpu().numpy()
    for i, (got, want) in enumerate(zip(rows(res), case["trials"])):
        assert got == (want["events"], want["objects"], want["t_end"], want["sum_wait"], want["counters8"]), (engine, name, i)
        assert trace_digest(tk[i], tt[i], got[0]) == want["trace_sha256"], (engine, name, i, "pop trace")


def per_trial_case():
    i = np.arange(N)
    arr = np.array([UP[k % 7] for k in i], dtype=np.float64)
    srv = np.array([REPAIR[k % 5] for k in i], dtype=np.float64)
    assert not (srv == 1.0).any()
    return {"servers": 5, "num_objects": 300, "params": [8, 0]}, arr, srv


def test_per_trial_parameters_static_equals_general_equals_the_reference(libs):
    """197 trials from first_trial 4093, each warp mixing up times and repair times: each trial equals the reference run
    alone at its own parameters, and the static tier's answer equals the general engine's."""
    case, arr, srv = per_trial_case()
    got = {}
    for engine in ("static", "general"):
        res, repaired = launch(libs[engine], arr, srv, case, first=FIRST, trace=0)
        assert repaired == 0 and (res.status.cpu().numpy() == 0).all(), engine
        got[engine] = rows(res)
    assert got["static"] == got["general"]
    assert len({r[0] for r in got["static"][:32]}) > 16          # the trials of a warp differ
    ref = load_repair_ref()
    if ref is None:
        pytest.skip("oracle/_ref/librepairdrv.so did not travel with this snapshot")
    for i in range(N):
        w = ref_run(ref, case["servers"], MASTER, FIRST + i, 1, case["num_objects"], float(arr[i]), float(srv[i]), case["params"])[0]
        want = (w.events, w.objects, float(w.t_end).hex(), float(w.sum_wait).hex(), list(w.counter))
        assert got["static"][i] == want, i


def test_host_buffer_entry_equals_the_device_entry(libs):
    """cimba_run_experiment over a host array with a counters field: the same trials as launch_trials, on both libraries;
    one in-tier case and one the static tier hands on."""
    dt = np.dtype([("arr_mean", "<f8"), ("srv_mean", "<f8"), ("obj_cnt", "<u8"), ("sum_wait", "<f8"), ("events", "<u8"),
                   ("t_end", "<f8"), ("status", "<u4"), ("pad", "<u4"), ("counters", "<u8", (8,))])
    for case, arr, srv in (per_trial_case(), (CASES["exit_holding"], None, None)):
        if arr is None:
            n = len(case["trials"])
            arr = np.full(n, float.fromhex(case["arr_mean"]))
            srv = np.full(n, float.fromhex(case["srv_mean"]))
        for engine in ("static", "general"):
            dev, _ = launch(libs[engine], arr, srv, case, first=FIRST, trace=0)
            exp = np.zeros(len(arr), dtype=dt)
            exp["arr_mean"], exp["srv_mean"] = arr, srv
            cb.cimba_run_experiment(exp, model=libs[engine], num_objects=case["num_objects"], master_seed=MASTER,
                                    first_trial=FIRST, servers=case["servers"], params=case["params"])
            assert not exp["status"].any()
            host = [(int(e["events"]), int(e["obj_cnt"]), float(e["t_end"]).hex(), float(e["sum_wait"]).hex(),
                     [int(v) for v in e["counters"]]) for e in exp]
            assert host == rows(dev), engine
