"""GPU tests of the static tier's second form (cimba_b200/csrc/cmb_static.cuh with static_interrupts: priorities, interrupts,
pre-emption) through the library's built-in routes: CIMBA_B200_VARIANT_STATIC on models 14 (ToolT, test/test_resource.c),
18 (CheeseT, test/test_resourcepool.c) and 21 (Tutorial2T, tutorial/tut_2_1.c).  Each must reproduce the unmodified reference bit
for bit - the vectors of tests/golden/cmb_engine_vectors.json with their pop traces, the golden files resource.txt and
resourcepool.txt, all 32 trials of tutorial 2's vectors - with diag[2] == 0: the tier answered, not the repair pass behind it.
The default routes of the three models are unchanged; the static route is compared with the general engine's on drawn
parameters and through the host-buffer entry."""
import json
import struct
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from cmb_cases import GOLD, MASTER, RESOURCEPOOL_GOLDEN_LINE, TRACE, case_id, check_trial, inverse_fmix64, wtdsummary_line

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
CASES = [c for c in GOLD["cases"] if c["model"] in (14, 18)]
TUT2 = json.loads((ROOT / "tests/golden/tutorial2_vectors.json").read_text())
STA, GEN = cb.VARIANT_STATIC, cb.VARIANT_GENERAL


def launch(model, n, *, servers, num_objects, master=MASTER, first=0, variant=STA, trace=0, arr=1.0, srv=1.0):
    dev = torch.device("cuda", torch.cuda.current_device())
    arr = torch.as_tensor(np.broadcast_to(np.asarray(arr, dtype=np.float64), (n,)).copy(), device=dev)
    srv = torch.as_tensor(np.broadcast_to(np.asarray(srv, dtype=np.float64), (n,)).copy(), device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(arr, srv, num_objects=num_objects, master_seed=master, first_trial=first, model=model, servers=servers,
                           trace_cap=trace, variant=variant, diag=diag)
    torch.cuda.synchronize()
    return res, int(diag[2].item())


def rows(res):
    cnt = res.counters.cpu().numpy().astype(np.uint64)
    return [(int(e), int(o), float(t).hex(), float(s).hex(), [int(v) for v in c])
            for e, o, t, s, c in zip(res.events.cpu().numpy().astype(np.uint64), res.objects.cpu().numpy().astype(np.uint64),
                                     res.t_end.cpu().numpy(), res.sum_wait.cpu().numpy(), cnt)]


def _double(u):
    return struct.unpack("<d", struct.pack("<Q", int(u) & (2**64 - 1)))[0]


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
                    max_queue=mq[i] if case["model"] == 14 else None)


def test_static_route_reproduces_the_resource_golden_file():
    """test/reference/resource.txt: history N 30, mean 0.9816, Target_3 pre-empted at t = 6.3280, 85 events."""
    res, repaired = launch(cb.MODEL_RESOURCE_RECORDED, 1, servers=1, num_objects=25, master=inverse_fmix64(0x34F05C64D7AD598F))
    c = [int(v) for v in res.counters.cpu().numpy().astype(np.uint64)[0]]
    assert repaired == 0 and int(res.status[0]) == 0 and int(res.events[0]) == 85 and int(res.max_queue[0]) == 30
    assert "%.4f" % _double(c[3]) == "0.9816" and "%.4f" % _double(c[4]) == "6.3280" and c[5] == 3 and c[1] == 1


def test_static_route_reproduces_the_resourcepool_golden_file():
    """test/reference/resourcepool.txt: the reference's seed, 20 units, 100 time units, the file's summary line."""
    res, repaired = launch(cb.MODEL_POOL_RECORDED, 1, servers=20, num_objects=100, master=inverse_fmix64(0x34F05C64D7AD598F))
    c = [int(v) for v in res.counters.cpu().numpy().astype(np.uint64)[0]]
    assert repaired == 0 and int(res.status[0]) == 0 and c[0] == 120
    assert wtdsummary_line(cb.lib, c) == RESOURCEPOOL_GOLDEN_LINE


def test_second_tutorial_on_the_static_route_matches_all_vector_trials():
    """All 32 trials of tutorial 2's vectors (about 660 000 events each): events, final clock, the stream's next raw output."""
    n = len(TUT2["trials"])
    res, repaired = launch(cb.MODEL_TUTORIAL2, n, servers=1, num_objects=0, master=TUT2["master"])
    assert repaired == 0 and (res.status.cpu().numpy() == 0).all()
    ev, te, cnt = res.events.cpu().tolist(), res.t_end.cpu().tolist(), res.counters.cpu().numpy()
    for i, want in enumerate(TUT2["trials"]):
        assert (ev[i], float(te[i]).hex(), int(cnt[i][0]) & (2**64 - 1)) == (want["events"], want["t_end"], want["next_raw"]), i


@pytest.mark.parametrize("model", [cb.MODEL_RESOURCE_RECORDED, cb.MODEL_POOL_RECORDED])
def test_static_route_equals_the_general_engine_on_drawn_parameters(model):
    """Three hundred trials per parameter set, from an odd first trial, at drawn capacities and durations: the static route and
    the general engine give the same rows, and the tier answers every trial itself."""
    rnd = np.random.default_rng(20261015 + model)
    for _ in range(3):
        servers, nobj, first = int(rnd.integers(1, 41)), int(rnd.integers(20, 400)), int(rnd.integers(0, 100_000))
        got = {}
        for variant in (STA, GEN):
            res, repaired = launch(model, 300, servers=servers, num_objects=nobj, first=first, variant=variant)
            assert repaired == 0 and (res.status.cpu().numpy() == 0).all(), (variant, servers, nobj)
            got[variant] = rows(res)
        assert got[STA] == got[GEN], (model, servers, nobj, first)
        assert len({r[0] for r in got[STA][:32]}) > 16          # the trials of a warp differ


def test_host_buffer_entry_equals_the_device_entry_for_the_pool_model():
    """cimba_b200_run_experiment over a host array with a counters field, model 18 on VARIANT_STATIC: the same rows as
    launch_trials."""
    n, servers, nobj, first = 197, 13, 150, 4093
    dev, repaired = launch(cb.MODEL_POOL_RECORDED, n, servers=servers, num_objects=nobj, first=first)
    assert repaired == 0
    dt = np.dtype([("arr_mean", "<f8"), ("srv_mean", "<f8"), ("obj_cnt", "<u8"), ("sum_wait", "<f8"), ("events", "<u8"),
                   ("t_end", "<f8"), ("status", "<u4"), ("pad", "<u4"), ("counters", "<u8", (8,))])
    exp = np.zeros(n, dtype=dt)
    exp["arr_mean"], exp["srv_mean"] = 1.0, 1.0
    cb.cimba_run_experiment(exp, model=cb.MODEL_POOL_RECORDED, num_objects=nobj, master_seed=MASTER, first_trial=first,
                            servers=servers, variant=STA)
    assert not exp["status"].any()
    host = [(int(e["events"]), int(e["obj_cnt"]), float(e["t_end"]).hex(), float(e["sum_wait"]).hex(), [int(v) for v in e["counters"]])
            for e in exp]
    assert host == rows(dev)
