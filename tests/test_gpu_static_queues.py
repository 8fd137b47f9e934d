"""GPU tests of the static tier's cmb_priorityqueue and cmb_condition (cimba_b200/csrc/cmb_static.cuh) through the library's
built-in routes: CIMBA_B200_VARIANT_STATIC on models 3 and 11 (GuardedT, test/test_objectqueue.c), 13 (test/test_priorityqueue.c)
and 6 (QueueAndTideT).  Each must reproduce the unmodified reference bit for bit - the vectors of tests/golden/cmb_engine_vectors.json
with their pop traces, the golden files objectqueue.txt and priorityqueue.txt - with diag[2] == 0: the tier answered, not the
repair pass behind it.  The default routes of the four models are unchanged; the static route is compared with the general
engine's and the default route's on drawn and per-trial parameters, through the host-buffer entry, and above the tier's tables,
where the repair pass must answer."""
import json
import struct
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from cmb_cases import GOLD, MASTER, TRACE, case_id, check_trial, inverse_fmix64

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
MODELS = (cb.MODEL_GUARDED, cb.MODEL_PRIOQ, cb.MODEL_GUARDED_RECORDED, cb.MODEL_PRIOQ_RECORDED)
CASES = [c for c in GOLD["cases"] if c["model"] in MODELS]
STA, GEN = cb.VARIANT_STATIC, cb.VARIANT_GENERAL
KAT_SEED = 0x34F05C64D7AD598F


def launch(model, n, *, servers, num_objects, master=MASTER, first=0, variant=STA, trace=0, arr=1.0, srv=1.0):
    dev = torch.device("cuda", torch.cuda.current_device())
    arr = torch.as_tensor(np.broadcast_to(np.asarray(arr, dtype=np.float64), (n,)).copy(), device=dev)
    srv = torch.as_tensor(np.broadcast_to(np.asarray(srv, dtype=np.float64), (n,)).copy(), device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(arr, srv, num_objects=num_objects, master_seed=master, first_trial=first, model=model, servers=servers,
                           trace_cap=trace, variant=variant, diag=diag)
    torch.cuda.synchronize()
    return res, int(diag[2].item())


def rows(res, max_queue=True):
    cnt = res.counters.cpu().numpy().astype(np.uint64)
    mq = res.max_queue.cpu().numpy() if max_queue else [0] * len(cnt)
    return [(int(e), int(o), float(t).hex(), float(s).hex(), int(q), [int(v) for v in c])
            for e, o, t, s, q, c in zip(res.events.cpu().numpy().astype(np.uint64), res.objects.cpu().numpy().astype(np.uint64),
                                        res.t_end.cpu().numpy(), res.sum_wait.cpu().numpy(), mq, cnt)]


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_static_route_matches_the_reference_vectors(case):
    n = len(case["trials"])
    res, repaired = launch(case["model"], n, servers=case["servers"], num_objects=case["num_objects"], trace=TRACE,
                           arr=float.fromhex(case["arr_mean"]), srv=float.fromhex(case["srv_mean"]))
    assert repaired == 0
    assert (res.status.cpu().numpy() == 0).all(), res.status.cpu().numpy()
    tk, tt = res.trace_key.cpu().numpy(), res.trace_time.cpu().numpy()
    cnt, mq = res.counters.cpu().numpy().astype(np.uint64), res.max_queue.cpu().numpy()
    ev, ob, te, sw = (res.events.cpu().numpy(), res.objects.cpu().numpy(), res.t_end.cpu().numpy(), res.sum_wait.cpu().numpy())
    for i, want in enumerate(case["trials"]):
        assert [int(v) for v in cnt[i]] == want["counters8"], (i, "all eight counters")
        check_trial(want, ev[i], ob[i], te[i], sw[i], [int(v) for v in cnt[i]], tk[i], tt[i], f"trial {i}",
                    max_queue=mq[i] if case["model"] in (11, 13) else None)
        if case["model"] in (3, 6):
            assert int(mq[i]) == want["max_fel"], (i, "fel_high")


@pytest.mark.parametrize("model", [cb.MODEL_GUARDED_RECORDED, cb.MODEL_PRIOQ_RECORDED])
def test_static_route_reproduces_the_queue_golden_files(model):
    """test/reference/objectqueue.txt and priorityqueue.txt: the reference's seed, capacity 10, 10^6 time units (8.46 million
    events in one lane): history N 5689021, mean 5.008, every word equal to the reference's record."""
    gold = json.loads((ROOT / "tests/golden/reference_vectors.json").read_text())
    want = [t for t in gold["trials"] if t["model"] == model and t["num_objects"] == 1_000_000][0]
    res, repaired = launch(model, 1, servers=10, num_objects=1_000_000, master=inverse_fmix64(KAT_SEED))
    c = [int(v) for v in res.counters.cpu().numpy().astype(np.uint64)[0]]
    mean = struct.unpack("<d", struct.pack("<Q", c[6]))[0]
    assert repaired == 0 and int(res.status[0]) == 0
    assert int(res.max_queue[0]) == 5689021 and "%.4g" % mean == "5.008"
    assert c == want["counters"]
    assert (int(res.events[0]), int(res.objects[0])) == (want["events"], want["objects"])
    assert float(res.t_end[0]).hex() == want["t_end"] and float(res.sum_wait[0]).hex() == want["sum_wait"]


@pytest.mark.parametrize("model", MODELS)
def test_static_route_equals_the_general_engine_on_drawn_parameters(model):
    """Three hundred trials per parameter set, from an odd first trial, at drawn capacities within the tier's tables and
    durations: the static route and the general engine give the same rows, and the tier answers every trial itself."""
    rnd = np.random.default_rng(20261016 + model)
    top = 16 if model in (cb.MODEL_GUARDED, cb.MODEL_GUARDED_RECORDED) else 15
    for _ in range(3):
        servers, nobj, first = int(rnd.integers(1, top + 1)), int(rnd.integers(50, 800)), int(rnd.integers(0, 100_000)) | 1
        got = {}
        for variant in (STA, GEN):
            res, repaired = launch(model, 300, servers=servers, num_objects=nobj, first=first, variant=variant)
            assert repaired == 0 and (res.status.cpu().numpy() == 0).all(), (variant, servers, nobj)
            got[variant] = rows(res)
        assert got[STA] == got[GEN], (model, servers, nobj, first)
        assert len({r[0] for r in got[STA][:32]}) > 16          # the trials of a warp differ


@pytest.mark.parametrize("model", MODELS)
def test_per_trial_means_agree_on_all_three_routes(model):
    """197 trials from first_trial 4093, each with its own arr_mean and srv_mean: the static route, the general engine and the
    default route (the fixed-capacity kernel with its repair pass) give the same rows."""
    n, first, servers, nobj = 197, 4093, 9, 400
    rnd = np.random.default_rng(4093 + model)
    arr, srv = rnd.uniform(0.4, 1.6, n), rnd.uniform(0.5, 1.5, n)
    got = {}
    for variant in (STA, GEN, 0):
        res, repaired = launch(model, n, servers=servers, num_objects=nobj, first=first, variant=variant, arr=arr, srv=srv)
        assert (res.status.cpu().numpy() == 0).all(), variant
        if variant == STA:
            assert repaired == 0
        got[variant] = rows(res, max_queue=variant != 0)
    assert got[STA] == got[GEN]
    assert [r[:4] + r[5:] for r in got[STA]] == [r[:4] + r[5:] for r in got[0]]


def test_host_buffer_entry_equals_the_device_entry_for_the_priority_queue_model():
    """cimba_b200_run_experiment over a host array with a counters field, model 13 on VARIANT_STATIC: the same rows as
    launch_trials."""
    n, servers, nobj, first = 197, 7, 300, 4093
    dev, repaired = launch(cb.MODEL_PRIOQ_RECORDED, n, servers=servers, num_objects=nobj, first=first)
    assert repaired == 0
    dt = np.dtype([("arr_mean", "<f8"), ("srv_mean", "<f8"), ("obj_cnt", "<u8"), ("sum_wait", "<f8"), ("events", "<u8"),
                   ("t_end", "<f8"), ("status", "<u4"), ("pad", "<u4"), ("counters", "<u8", (8,))])
    exp = np.zeros(n, dtype=dt)
    exp["arr_mean"], exp["srv_mean"] = 1.0, 1.0
    cb.cimba_run_experiment(exp, model=cb.MODEL_PRIOQ_RECORDED, num_objects=nobj, master_seed=MASTER, first_trial=first,
                            servers=servers, variant=STA)
    assert not exp["status"].any()
    host = [(int(e["events"]), int(e["obj_cnt"]), float(e["t_end"]).hex(), float(e["sum_wait"]).hex(), [int(v) for v in e["counters"]])
            for e in exp]
    assert host == [r[:4] + r[5:] for r in rows(dev)]


@pytest.mark.parametrize("model", MODELS)
def test_above_the_tiers_tables_the_repair_pass_answers(model):
    """Capacity 40 in heavy traffic: the priority queue outgrows its 16-entry table, the object queue its 32-entry window.  Those
    trials are re-run by the general engine inside the same launch (diag[2] > 0), and the rows equal the general engine's."""
    n, nobj, first = 256, 2000, 77
    got, repaired = {}, {}
    for variant in (STA, GEN):
        res, repaired[variant] = launch(model, n, servers=40, num_objects=nobj, first=first, variant=variant, arr=0.5)
        assert (res.status.cpu().numpy() == 0).all(), variant
        got[variant] = rows(res)
    assert repaired[STA] > 0 and repaired[GEN] == 0
    assert got[STA] == got[GEN]
