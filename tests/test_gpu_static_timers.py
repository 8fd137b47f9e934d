"""GPU tests of the static tier's timers, resume / yield, waits on processes and events, the model's events by handle and observers
(cimba_b200/csrc/cmb_static.cuh) through the library's route CIMBA_B200_VARIANT_STATIC on model 8 (FrontDeskT).  It must reproduce
the unmodified reference bit for bit - the vectors of tests/golden/cmb_engine_vectors.json with their pop traces - with diag[2] == 0:
the tier answered, not the repair pass behind it.  It must also agree with the plain-C port of the reference, with the general
engine on drawn sets, with the general engine and the default route (timers_kernel and its repair pass) on per-trial means, and
through the host-buffer entry."""
import numpy as np
import pytest
import torch

import cimba_b200 as cb
from cmb_cases import GOLD, MASTER, TRACE, case_id, check_trial

pytestmark = pytest.mark.gpu
CASES = [c for c in GOLD["cases"] if c["model"] == cb.MODEL_TIMERS]
STA, GEN = cb.VARIANT_STATIC, cb.VARIANT_GENERAL
KAT_SEED = 0x34F05C64D7AD598F


def launch(n, *, num_objects, master=MASTER, first=0, variant=STA, trace=0, arr=1.0, srv=1.0):
    dev = torch.device("cuda", torch.cuda.current_device())
    arr = torch.as_tensor(np.broadcast_to(np.asarray(arr, dtype=np.float64), (n,)).copy(), device=dev)
    srv = torch.as_tensor(np.broadcast_to(np.asarray(srv, dtype=np.float64), (n,)).copy(), device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(arr, srv, num_objects=num_objects, master_seed=master, first_trial=first, model=cb.MODEL_TIMERS, servers=1,
                           trace_cap=trace, variant=variant, diag=diag)
    torch.cuda.synchronize()
    return res, int(diag[2].item())


def counters(res):
    return np.ascontiguousarray(res.counters.cpu().numpy(), dtype=np.int64).view(np.uint64)


def rows(res, max_queue=True):
    cnt = counters(res)
    mq = res.max_queue.cpu().numpy() if max_queue else [0] * len(cnt)
    return [(int(e), int(o), float(t).hex(), float(s).hex(), int(q), [int(v) for v in c])
            for e, o, t, s, q, c in zip(res.events.cpu().numpy().astype(np.uint64), res.objects.cpu().numpy().astype(np.uint64),
                                        res.t_end.cpu().numpy(), res.sum_wait.cpu().numpy(), mq, cnt)]


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_static_route_matches_the_reference_vectors(case):
    n = len(case["trials"])
    res, repaired = launch(n, num_objects=case["num_objects"], trace=TRACE, arr=float.fromhex(case["arr_mean"]),
                           srv=float.fromhex(case["srv_mean"]))
    assert repaired == 0
    assert (res.status.cpu().numpy() == 0).all(), res.status.cpu().numpy()
    tk, tt = res.trace_key.cpu().numpy(), res.trace_time.cpu().numpy()
    cnt, mq = counters(res), res.max_queue.cpu().numpy()
    ev, ob, te, sw = (res.events.cpu().numpy(), res.objects.cpu().numpy(), res.t_end.cpu().numpy(), res.sum_wait.cpu().numpy())
    for i, want in enumerate(case["trials"]):
        assert [int(v) for v in cnt[i]] == want["counters8"], (i, "all eight counters")
        check_trial(want, ev[i], ob[i], te[i], sw[i], [int(v) for v in cnt[i]], tk[i], tt[i], f"trial {i}")
        assert int(mq[i]) == want["max_fel"], (i, "fel_high")


@pytest.mark.parametrize("dur,am,sm", [(500, 1.0, 0.6), (300, 0.4, 1.2), (200, 2.0, 0.3), (1, 1.0, 1.0), (3, 1.0, 1.0)])
def test_static_route_matches_the_port(port, dur, am, sm):
    """96 trials at the durations and means of the general engine's parity test: the plain-C port's events, objects, clock, sums,
    counters and fel_high, every trial answered by the tier or (for a trial that needs more spare slots) its repair pass."""
    from oracle_libs import run_trials
    n = 96
    res, _ = launch(n, num_objects=dur, master=KAT_SEED, arr=am, srv=sm)
    want = run_trials(port, "port", cb.MODEL_TIMERS, 1, KAT_SEED, 0, n, dur, am, sm)
    assert (res.status.cpu().numpy() == 0).all()
    got = rows(res)
    for i, w in enumerate(want):
        assert got[i] == (w.events, w.objects, float(w.t_end).hex(), float(w.sum_wait).hex(), w.max_fel, w.counters()), i


def test_static_route_equals_the_general_engine_on_drawn_parameters():
    """Three hundred trials per parameter set, from an odd first trial, at drawn durations and means: the static route and the
    general engine give the same rows, and the tier answers nearly all of them itself."""
    rnd = np.random.default_rng(20261016 + cb.MODEL_TIMERS)
    for _ in range(3):
        nobj, first = int(rnd.integers(50, 800)), int(rnd.integers(0, 100_000)) | 1
        am, sm = float(rnd.choice([0.4, 0.8, 1.0, 2.0])), float(rnd.choice([0.3, 0.6, 1.0, 1.2]))
        got, repaired = {}, {}
        for variant in (STA, GEN):
            res, repaired[variant] = launch(300, num_objects=nobj, first=first, variant=variant, arr=am, srv=sm)
            assert (res.status.cpu().numpy() == 0).all(), (variant, nobj, am, sm)
            got[variant] = rows(res)
        assert got[STA] == got[GEN], (nobj, am, sm, first)
        assert repaired[GEN] == 0 and repaired[STA] <= 15, repaired
        assert len({r[0] for r in got[STA][:32]}) > 16          # the trials of a warp differ


def test_a_trial_that_needs_a_ninth_spare_slot_is_answered_by_the_repair_pass():
    """512 trials of 1000 time units: a few have nine engine and model events pending at once, one more than the route's spare
    slots.  The tier flags them, the general engine re-runs them inside the same launch (diag[2] > 0), and the rows equal the
    general engine's."""
    got, repaired = {}, {}
    for variant in (STA, GEN):
        res, repaired[variant] = launch(512, num_objects=1000, first=77, variant=variant, arr=0.8, srv=1.0)
        assert (res.status.cpu().numpy() == 0).all(), variant
        got[variant] = rows(res)
    assert repaired[STA] > 0 and repaired[GEN] == 0, repaired
    assert got[STA] == got[GEN]


def test_per_trial_means_agree_on_all_three_routes():
    """197 trials from first_trial 4093, each with its own arr_mean and srv_mean: the static route, the general engine and the
    default route (timers_kernel with its repair pass) give the same rows."""
    n, first, nobj = 197, 4093, 400
    rnd = np.random.default_rng(4093 + cb.MODEL_TIMERS)
    arr, srv = rnd.uniform(0.4, 1.6, n), rnd.uniform(0.5, 1.5, n)
    got = {}
    for variant in (STA, GEN, 0):
        res, _ = launch(n, num_objects=nobj, first=first, variant=variant, arr=arr, srv=srv)
        assert (res.status.cpu().numpy() == 0).all(), variant
        got[variant] = rows(res)
    assert got[STA] == got[GEN] == got[0]


def test_host_buffer_entry_equals_the_device_entry():
    """cimba_b200_run_experiment over a host array with a counters field, model 8 on VARIANT_STATIC: the same rows as
    launch_trials."""
    n, nobj, first = 197, 300, 4093
    dev, repaired = launch(n, num_objects=nobj, first=first)
    dt = np.dtype([("arr_mean", "<f8"), ("srv_mean", "<f8"), ("obj_cnt", "<u8"), ("sum_wait", "<f8"), ("events", "<u8"),
                   ("t_end", "<f8"), ("status", "<u4"), ("pad", "<u4"), ("counters", "<u8", (8,))])
    exp = np.zeros(n, dtype=dt)
    exp["arr_mean"], exp["srv_mean"] = 1.0, 1.0
    cb.cimba_run_experiment(exp, model=cb.MODEL_TIMERS, num_objects=nobj, master_seed=MASTER, first_trial=first, servers=1,
                            variant=STA)
    assert not exp["status"].any()
    host = [(int(e["events"]), int(e["obj_cnt"]), float(e["t_end"]).hex(), float(e["sum_wait"]).hex(), [int(v) for v in e["counters"]])
            for e in exp]
    assert host == [r[:4] + r[5:] for r in rows(dev)]
