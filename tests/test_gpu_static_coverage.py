"""GPU tests of the last fixed-process coverage models on the static tier's second form (cimba_b200/csrc/cmb_static.cuh) through
the library's route CIMBA_B200_VARIANT_STATIC: model 4 (PoolFightT: a pool with priorities, pre-emption and interrupts), model 5
(WorkshopT<S, false>: a cmb_buffer with partial puts and gets, a resource with a pre-empting worker, a nuisance) and model 12
(WorkshopT<S, true>: test/test_buffer.c as it stands, the level history on).  They must reproduce the unmodified reference bit for
bit - the vectors of tests/golden/cmb_engine_vectors.json with their pop traces and test/reference/buffer.txt - with diag[2] == 0:
the tier answered, not the repair pass behind it.  They must also agree with the plain-C port of the reference, with the general
engine on drawn sets, with the general engine and the default route (preempt_kernel / buffer_kernel and their repair pass) on
per-trial means, and through the host-buffer entry."""
import struct

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from cmb_cases import GOLD, MASTER, TRACE, case_id, check_trial, inverse_fmix64

pytestmark = pytest.mark.gpu
MODELS = (cb.MODEL_PREEMPT, cb.MODEL_BUFFER, cb.MODEL_BUFFER_RECORDED)
CASES = [c for c in GOLD["cases"] if c["model"] in MODELS]
REPORTS_FEL = (cb.MODEL_PREEMPT, cb.MODEL_BUFFER)      # model 12 reports its history's sample count instead
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


def counters(res):
    return np.ascontiguousarray(res.counters.cpu().numpy(), dtype=np.int64).view(np.uint64)


def rows(res):
    return [(int(e), int(o), float(t).hex(), float(s).hex(), int(q), [int(v) for v in c])
            for e, o, t, s, q, c in zip(res.events.cpu().numpy().astype(np.uint64), res.objects.cpu().numpy().astype(np.uint64),
                                        res.t_end.cpu().numpy(), res.sum_wait.cpu().numpy(), res.max_queue.cpu().numpy(), counters(res))]


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_static_route_matches_the_reference_vectors(case):
    model, n = case["model"], len(case["trials"])
    res, repaired = launch(model, n, servers=case["servers"], num_objects=case["num_objects"], trace=TRACE,
                           arr=float.fromhex(case["arr_mean"]), srv=float.fromhex(case["srv_mean"]))
    assert repaired == 0
    assert (res.status.cpu().numpy() == 0).all(), res.status.cpu().numpy()
    tk, tt = res.trace_key.cpu().numpy(), res.trace_time.cpu().numpy()
    cnt, mq = counters(res), res.max_queue.cpu().numpy()
    ev, ob, te, sw = (res.events.cpu().numpy(), res.objects.cpu().numpy(), res.t_end.cpu().numpy(), res.sum_wait.cpu().numpy())
    for i, want in enumerate(case["trials"]):
        assert [int(v) for v in cnt[i]] == want["counters8"], (i, "all eight counters")
        check_trial(want, ev[i], ob[i], te[i], sw[i], [int(v) for v in cnt[i]], tk[i], tt[i], f"trial {i}")
        if model in REPORTS_FEL:
            assert int(mq[i]) == want["max_fel"], (i, "fel_high")


def test_static_route_reproduces_the_reference_buffer_golden_file():
    """test/reference/buffer.txt through the static route: the reference's seed, capacity 10, 10 000 time units, level history
    N 41876, time-weighted mean 4.980, answered by the tier itself."""
    res, repaired = launch(cb.MODEL_BUFFER_RECORDED, 1, servers=10, num_objects=10_000, master=inverse_fmix64(KAT_SEED))
    assert int(res.status[0]) == 0 and repaired == 0
    mean = struct.unpack("<d", struct.pack("<Q", int(counters(res)[0][4])))[0]
    assert int(res.max_queue[0]) == 41876 and "%.3f" % mean == "4.980"


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("cap,dur,am,sm", [(1, 300, 1.0, 1.0), (5, 500, 0.6, 1.2), (10, 200, 1.5, 0.5), (20, 400, 1.0, 1.0),
                                           (40, 3, 1.0, 1.0)])
def test_static_route_matches_the_port(port, model, cap, dur, am, sm):
    """96 trials at several capacities, durations and (for models 5 and 12) means: the plain-C port's events, objects, clock, sums,
    counters and max_queue, every trial answered by the tier or (for a trial that needs more spare slots) its repair pass."""
    from oracle_libs import run_trials
    n = 96
    if model == cb.MODEL_PREEMPT:
        am, sm = 1.0, 1.0
    res, _ = launch(model, n, servers=cap, num_objects=dur, master=KAT_SEED, arr=am, srv=sm)
    want = run_trials(port, "port", model, cap, KAT_SEED, 0, n, dur, am, sm)
    assert (res.status.cpu().numpy() == 0).all()
    got = rows(res)
    for i, w in enumerate(want):
        q = w.max_fel if model in REPORTS_FEL else w.max_queue
        assert got[i] == (w.events, w.objects, float(w.t_end).hex(), float(w.sum_wait).hex(), q, w.counters()), (model, cap, i)


@pytest.mark.parametrize("model", MODELS)
def test_static_route_equals_the_general_engine_on_drawn_parameters(model):
    """Three hundred trials per parameter set, from an odd first trial, at drawn capacities, durations and (for 5 and 12) means:
    the static route and the general engine give the same rows."""
    rnd = np.random.default_rng(20261016 + model)
    for _ in range(3):
        cap, nobj, first = int(rnd.integers(1, 41)), int(rnd.integers(50, 800)), int(rnd.integers(0, 100_000)) | 1
        am, sm = (1.0, 1.0) if model == cb.MODEL_PREEMPT else (float(rnd.choice([0.5, 1.0, 1.5])), float(rnd.choice([0.5, 1.0, 2.0])))
        got, repaired = {}, {}
        for variant in (STA, GEN):
            res, repaired[variant] = launch(model, 300, servers=cap, num_objects=nobj, first=first, variant=variant, arr=am, srv=sm)
            assert (res.status.cpu().numpy() == 0).all(), (variant, cap, nobj, am, sm)
            got[variant] = rows(res)
        assert got[STA] == got[GEN], (model, cap, nobj, am, sm, first)
        assert repaired[GEN] == 0 and repaired[STA] <= 30, repaired
        assert len({r[0] for r in got[STA][:32]}) > 16          # the trials of a warp differ


def test_a_pool_trial_that_needs_a_fifth_spare_slot_is_answered_by_the_repair_pass():
    """Model 4, 512 trials at capacity 10 and 500 time units: a few have a fifth engine or model event pending at once (a rat
    pre-empting several holders while the cat's interrupt and the end event wait), one more than the route's spare slots.  The
    tier flags them, the general engine re-runs them inside the same launch (diag[2] > 0), and the rows equal the general
    engine's."""
    got, repaired = {}, {}
    for variant in (STA, GEN):
        res, repaired[variant] = launch(cb.MODEL_PREEMPT, 512, servers=10, num_objects=500, first=77, variant=variant)
        assert (res.status.cpu().numpy() == 0).all(), variant
        got[variant] = rows(res)
    assert repaired[STA] > 0 and repaired[GEN] == 0, repaired
    assert got[STA] == got[GEN]


@pytest.mark.parametrize("model", [cb.MODEL_BUFFER, cb.MODEL_BUFFER_RECORDED])
def test_per_trial_means_agree_on_all_three_routes(model):
    """197 trials from first_trial 4093, each with its own arr_mean and srv_mean: the static route, the general engine and the
    default route (buffer_kernel with its repair pass) give the same rows."""
    n, first, nobj = 197, 4093, 400
    rnd = np.random.default_rng(4093 + model)
    arr, srv = rnd.uniform(0.4, 1.6, n), rnd.uniform(0.5, 1.5, n)
    got = {}
    for variant in (STA, GEN, 0):
        res, _ = launch(model, n, servers=10, num_objects=nobj, first=first, variant=variant, arr=arr, srv=srv)
        assert (res.status.cpu().numpy() == 0).all(), variant
        got[variant] = rows(res)
    assert got[STA] == got[GEN] == got[0]


@pytest.mark.parametrize("model", MODELS)
def test_host_buffer_entry_equals_the_device_entry(model):
    """cimba_b200_run_experiment over a host array with a counters field on VARIANT_STATIC: the same rows as launch_trials."""
    n, nobj, first = 197, 300, 4093
    dev, _ = launch(model, n, servers=10, num_objects=nobj, first=first)
    dt = np.dtype([("arr_mean", "<f8"), ("srv_mean", "<f8"), ("obj_cnt", "<u8"), ("sum_wait", "<f8"), ("events", "<u8"),
                   ("t_end", "<f8"), ("status", "<u4"), ("pad", "<u4"), ("counters", "<u8", (8,))])
    exp = np.zeros(n, dtype=dt)
    exp["arr_mean"], exp["srv_mean"] = 1.0, 1.0
    cb.cimba_run_experiment(exp, model=model, num_objects=nobj, master_seed=MASTER, first_trial=first, servers=10, variant=STA)
    assert not exp["status"].any()
    host = [(int(e["events"]), int(e["obj_cnt"]), float(e["t_end"]).hex(), float(e["sum_wait"]).hex(), [int(v) for v in e["counters"]])
            for e in exp]
    assert host == [r[:4] + r[5:] for r in rows(dev)]
