"""The on-chip queue window of mm1_kernel (MODEL_MM1, variant 0): MM1_WINDOW = 48 stamps per trial in shared memory, the
rest in the trial's HBM ring of queue_spill_cap entries; a put past both voids the trial and the repair pass re-runs it.  The
window is a ring whose head and tail advance by a compare-free wrap (mm1_fast.cuh), so its edges are tested where they are:
queues that peak exactly at 47, 48, 49 and 50 entries, queues that cross 48 many times, and the overflow edge at
48 + queue_spill_cap and one past it.

Each trial's means are picked by running the oracle on the CPU here, so that its queue peaks where the case needs it.
Everything is compared bit for bit with the oracle run alone at each trial's own parameters: events, objects, t_end,
sum_wait and status, max_queue where the trial did not need the repair pass, and full pop traces where the case is small;
and with variant 1 (queue_kernel<0>, a 32-entry window) on the trials it runs clean."""
import numpy as np
import pytest
import torch

import cimba_b200 as cb
from oracle_libs import load_port, run_trials, trace_trial

pytestmark = pytest.mark.gpu

MASTER = 0x6A09E667F3BCC909
FIRST = 4099
WINDOW = 48                             # mm1_fast.cuh MM1_WINDOW
RING = 512                              # the default queue_spill_cap
SCALES = (1.0, 0.37, 3.7)               # service means; the arrival mean is scale / rho
IDLE_RHO = 0.05


def _rho_grid(lo, hi, n):
    return [lo + (hi - lo) * k / (n - 1) for k in range(n)]


def _pick(port, n, nobj, edge, grid):
    """Per trial i < n: means (arr, srv) at which the oracle's run of trial FIRST + i peaks at edge[i % len(edge)], or else
    at another peak of `edge`; every 8th trial, and one the grid cannot place, is idle."""
    out = []
    for i in range(n):
        scale = SCALES[i % len(SCALES)]
        out.append((scale / IDLE_RHO, scale))
        if i % 8 == 7:
            continue
        want = edge[i % len(edge)]
        other = None
        for rho in grid:
            peak = run_trials(port, "port", 0, 1, MASTER, FIRST + i, 1, nobj, scale / rho, scale)[0].max_queue
            if peak == want:
                out[i] = (scale / rho, scale)
                break
            if other is None and peak in edge:
                other = (scale / rho, scale)
        else:
            if other is not None:
                out[i] = other
    return tuple(zip(*out))


def _launch(arr, srv, nobj, variant=0, trace=0, spill_cap=0, diag=None):
    dev = torch.device("cuda", torch.cuda.current_device())
    a = torch.tensor(arr, dtype=torch.float64, device=dev)
    s = torch.tensor(srv, dtype=torch.float64, device=dev)
    res = cb.launch_trials(a, s, num_objects=nobj, master_seed=MASTER, first_trial=FIRST, model=cb.MODEL_MM1,
                           mapping=cb.MAP_LANE, trace_cap=trace, variant=variant, queue_spill_cap=spill_cap, diag=diag)
    torch.cuda.synchronize(dev)
    out = {k: getattr(res, k).cpu().numpy().copy() for k in ("events", "objects", "status", "max_queue")}
    for k in ("t_end", "sum_wait"):
        out[k] = np.ascontiguousarray(getattr(res, k).cpu().numpy(), dtype=np.float64).view(np.uint64).copy()
    if trace:
        out["trace_key"] = res.trace_key.cpu().numpy().copy()
        out["trace_time"] = np.ascontiguousarray(res.trace_time.cpu().numpy(), dtype=np.float64).view(np.uint64).copy()
    return out


def _bits(x):
    return int(np.float64(x).view(np.uint64))


def _oracle(port, arr, srv, nobj):
    return [run_trials(port, "port", 0, 1, MASTER, FIRST + i, 1, nobj, float(arr[i]), float(srv[i]))[0]
            for i in range(len(arr))]


def _check_oracle(got, want, tag, spill_cap=RING):
    """max_queue only where the trial ran to its end in mm1_kernel: the repair pass's engine does not track it."""
    for i, w in enumerate(want):
        assert (int(got["events"][i]), int(got["objects"][i])) == (w.events, w.objects), (tag, i)
        assert int(got["t_end"][i]) == _bits(w.t_end) and int(got["sum_wait"][i]) == _bits(w.sum_wait), (tag, i)
        assert int(got["status"][i]) == 0, (tag, i, int(got["status"][i]))
        if w.max_queue <= WINDOW + spill_cap:
            assert int(got["max_queue"][i]) == w.max_queue, (tag, i, int(got["max_queue"][i]), w.max_queue)


def _check_trace(port, got, arr, srv, nobj, cap, tag):
    for i in range(len(arr)):
        r, keys, times = trace_trial(port, "port", 0, 1, cb.fmix64(MASTER, FIRST + i), nobj, float(arr[i]), float(srv[i]), cap)
        n = len(keys)
        assert n == min(cap, r.events), (tag, i)
        assert got["trace_key"][i, :n].tolist() == keys, (tag, i)
        assert got["trace_time"][i, :n].tolist() == [_bits(t) for t in times], (tag, i)


def _check_clean_variant1(v0, v1, tag):
    clean = [i for i in range(len(v0["events"])) if int(v1["status"][i]) == 0]
    assert clean, tag
    for k in v1:
        assert np.array_equal(v0[k][clean], v1[k][clean]), (tag, k)


def test_peaks_at_the_window_edge():
    """Two warps: trials whose queues peak at exactly 47, 48, 49 and 50 entries next to idle lanes; lanes park on the
    ziggurat's slow path as their streams have it.  Full pop traces, and variant 1 (all of them clean at these peaks)."""
    port = load_port()
    n, nobj = 64, 2000
    edge = (WINDOW - 1, WINDOW, WINDOW + 1, WINDOW + 2)
    arr, srv = _pick(port, n, nobj, edge, _rho_grid(0.85, 1.25, 201))
    want = _oracle(port, arr, srv, nobj)
    for t in edge:
        assert sum(1 for w in want if w.max_queue == t) >= 4, (t, [w.max_queue for w in want])
    cap = 4 * nobj + 8
    assert max(w.events for w in want) <= cap
    v0 = _launch(arr, srv, nobj, trace=cap)
    _check_oracle(v0, want, "variant 0")
    _check_trace(port, v0, arr, srv, nobj, cap, "variant 0")
    _check_clean_variant1(v0, _launch(arr, srv, nobj, variant=1, trace=cap), "variant 0 vs 1")


def test_crossing_the_window_many_times():
    """10^5 objects at rho = 0.99: queues pass 48 over and over, so the far path (puts into the HBM ring, refills of the
    window from it) runs many times per trial; one warp, idle and rho = 0.9 lanes in between.  A trial whose queue outgrows
    48 + 512 is re-run by the repair pass and must come back as the oracle has it too."""
    port = load_port()
    n, nobj = 32, 100_000
    rhos = [0.99 if i % 4 in (0, 1) else 0.9 if i % 4 == 2 else IDLE_RHO for i in range(n)]
    srv = [SCALES[i % 3] for i in range(n)]
    arr = [srv[i] / rhos[i] for i in range(n)]
    want = _oracle(port, arr, srv, nobj)
    assert sum(1 for w in want if WINDOW + 2 < w.max_queue <= WINDOW + RING) >= 8, [w.max_queue for w in want]
    diag = torch.zeros(4, dtype=torch.int64, device=torch.device("cuda", torch.cuda.current_device()))
    v0 = _launch(arr, srv, nobj, diag=diag)
    _check_oracle(v0, want, "variant 0")
    assert int(diag[2].item()) == sum(1 for w in want if w.max_queue > WINDOW + RING)
    _check_clean_variant1(v0, _launch(arr, srv, nobj, variant=1), "variant 0 vs 1")


@pytest.mark.parametrize("spill_cap", [16, 64])
def test_overflow_edge(spill_cap):
    """queue_spill_cap 16 and 64: a queue of 48 + cap entries still runs to the end in mm1_kernel, one more entry voids
    the trial and the repair pass re-runs it (diag[2] counts those).  Either way the result is the oracle's."""
    port = load_port()
    n, nobj = 64, 3000
    top = WINDOW + spill_cap
    edge = (top - 1, top, top + 1, top + 2)
    arr, srv = _pick(port, n, nobj, edge, _rho_grid(0.9, 1.6, 281))
    want = _oracle(port, arr, srv, nobj)
    for t in edge:
        assert sum(1 for w in want if w.max_queue == t) >= 2, (t, [w.max_queue for w in want])
    diag = torch.zeros(4, dtype=torch.int64, device=torch.device("cuda", torch.cuda.current_device()))
    v0 = _launch(arr, srv, nobj, spill_cap=spill_cap, diag=diag)
    _check_oracle(v0, want, f"variant 0, queue_spill_cap {spill_cap}", spill_cap)
    assert int(diag[2].item()) == sum(1 for w in want if w.max_queue > top)


@pytest.mark.parametrize("trace", [0, 1])
def test_eight_ctas_resident_per_sm(trace):
    """With the shared-memory carveout the library asks for, 8 CTAs of 64 lanes fit an SM: 65 536 trials in one wave."""
    assert cb.lib.cimba_b200_mm1_resident_ctas(trace) == 8, cb.lib.cimba_b200_last_error()
