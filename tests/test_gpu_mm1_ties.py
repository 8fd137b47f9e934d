"""Ties in time in mm1_kernel (MODEL_MM1, variant 0), the kernel bench.py measures.  The kernel keeps a trial's two pending
events in pop order and orders an inserted event with one strict compare, relying on the reference's tie-break (time
ascending, then key ascending) and on a new key being the largest issued so far.  A zero mean puts many events at the same
time, so the order is decided by the keys alone:

- both means 0: every event of the trial is at t = 0;
- the arrival mean 0 alone: every customer arrives at t = 0, fewer of them than the on-chip window holds, so the queue never
  leaves the window, and the server's wake-up ties with the arrivals' holds;
- the service mean 0 alone: every service ends at the moment it starts.

Lanes of these trials sit in one warp with ordinary ones (rho 0.9, 0.5 and 1.3).  Every trial is compared bit for bit with the
oracle run alone at its own parameters, pop for pop, and with variant 1 (queue_kernel<0>)."""
import numpy as np
import pytest
import torch

import cimba_b200 as cb
from oracle_libs import load_port, run_trials, trace_trial

pytestmark = pytest.mark.gpu

MASTER = 0x9E3779B97F4A7C15
FIRST = 31
WINDOW = 48                             # mm1_fast.cuh MM1_WINDOW
KINDS = ("both zero", "arrival zero", "service zero", "rho 0.9", "rho 0.5", "rho 1.3")


def _means(n):
    arr, srv = np.empty(n), np.empty(n)
    for i in range(n):
        kind = KINDS[i % len(KINDS)]
        s = 1.0 + 0.25 * (i % 3)
        arr[i], srv[i] = {"both zero": (0.0, 0.0), "arrival zero": (0.0, s), "service zero": (s, 0.0),
                          "rho 0.9": (s / 0.9, s), "rho 0.5": (s / 0.5, s), "rho 1.3": (s / 1.3, s)}[kind]
    return arr, srv


def _launch(arr, srv, nobj, variant, cap):
    dev = torch.device("cuda", torch.cuda.current_device())
    a = torch.tensor(arr, dtype=torch.float64, device=dev)
    s = torch.tensor(srv, dtype=torch.float64, device=dev)
    res = cb.launch_trials(a, s, num_objects=nobj, master_seed=MASTER, first_trial=FIRST, model=cb.MODEL_MM1,
                           trace_cap=cap, variant=variant)
    torch.cuda.synchronize(dev)
    out = {k: getattr(res, k).cpu().numpy() for k in ("events", "objects", "status", "max_queue", "trace_key")}
    for k in ("t_end", "sum_wait", "trace_time"):
        out[k] = np.ascontiguousarray(getattr(res, k).cpu().numpy(), dtype=np.float64).view(np.uint64)
    return out


def _bits(x):
    return int(np.float64(x).view(np.uint64))


@pytest.mark.parametrize("nobj", [1, 5, 40])
def test_ties_in_time_pop_for_pop(nobj):
    n = 3 * 32 + 7                      # three full warps and a partial one, every kind in every warp
    arr, srv = _means(n)
    cap = 4 * nobj + 8
    port = load_port()
    v0, v1 = _launch(arr, srv, nobj, 0, cap), _launch(arr, srv, nobj, 1, cap)
    for i in range(n):
        tag = (KINDS[i % len(KINDS)], i)
        w = run_trials(port, "port", 0, 1, MASTER, FIRST + i, 1, nobj, float(arr[i]), float(srv[i]))[0]
        assert (int(v0["events"][i]), int(v0["objects"][i])) == (w.events, w.objects), tag
        assert int(v0["t_end"][i]) == _bits(w.t_end) and int(v0["sum_wait"][i]) == _bits(w.sum_wait), tag
        assert int(v0["status"][i]) == 0 and int(v0["max_queue"][i]) == w.max_queue, tag
        if KINDS[i % len(KINDS)] == "arrival zero":
            assert w.max_queue >= nobj - 1 and w.max_queue < WINDOW, tag     # every customer queued at t = 0, on chip
        r, keys, times = trace_trial(port, "port", 0, 1, cb.fmix64(MASTER, FIRST + i), nobj, float(arr[i]),
                                     float(srv[i]), cap)
        k = len(keys)
        assert k == r.events <= cap, tag
        assert v0["trace_key"][i, :k].tolist() == keys, tag
        assert v0["trace_time"][i, :k].tolist() == [_bits(t) for t in times], tag
        if KINDS[i % len(KINDS)] == "both zero":
            assert all(t == 0.0 for t in times), tag
    for key in v0:
        assert np.array_equal(v0[key], v1[key]), key
