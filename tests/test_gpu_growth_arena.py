"""The general engine's growth arena at experiment scale, on the device: jobs whose trials together need more arena than the
workspace their route asks for (tests/arena_cases.py; the CPU checks those needs, with sanitizers, in tests/test_growth_arena.py).

* cimba_b200_launch flags and does not retry: every trial is either clean and bit-identical to reference arrays, or carries
  CIMBA_B200_TRIAL_ARENA_EXHAUSTED and nothing else; with the rings plus 1.25x the trials' summed need as workspace, none is.
* cimba_b200_run_experiment (and the all-GPU entry) re-runs what ran out with more workspace: rc 0, every row the reference's.

Reference arrays come from routes that never need the engine: the fast kernel or the static tier with HBM rings of 8192 entries,
where these queues peak below 6 000 (no trial repaired, diag[2] == 0).  M/M/c with 20 servers has no fast kernel; its reference is
the engine route with a workspace large enough that nothing is flagged, and the C port on a sample."""
import sys
import time
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from arena_cases import GPU_SHAPES, MASTER, estimated_need, rings_bytes, shape_of
from oracle_libs import load_port, run_trials

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
BIG_RING = 8192
FIELDS = ("events", "objects", "t_end", "sum_wait", "max_queue", "counters")


def _model_id(name):
    lib_model = GPU_SHAPES[name][0]
    if isinstance(lib_model, int):
        return lib_model
    sys.path.insert(0, str(ROOT / "scripts"))
    so = ROOT / "cimba_b200/lib/models" / f"lib{lib_model}.so"
    if not so.exists():
        import build_model
        build_model.build(ROOT / "examples" / f"{lib_model}.cu")
    return cb.load_model(so)


def _inputs(name):
    _, servers, trials, nobj, arr, srv = shape_of(name)
    dev = torch.device("cuda", torch.cuda.current_device())
    return (torch.full((trials,), arr, dtype=torch.float64, device=dev), torch.full((trials,), srv, dtype=torch.float64, device=dev),
            servers, nobj)


def _rows(res):
    torch.cuda.synchronize()
    return {f: getattr(res, f).cpu().numpy().copy() for f in FIELDS + ("status",)}


def _launch(name, model, variant, spill=0, workspace=None, diag=None):
    arr, srv, servers, nobj = _inputs(name)
    b = cb.TrialBuffers(arr.numel(), arr.device, 0, model, servers, variant, spill, nobj)
    if workspace is not None:
        b.workspace = torch.empty(workspace, dtype=torch.uint8, device=arr.device)
        b.workspace_bytes = workspace
    res = cb.launch_trials(arr, srv, num_objects=nobj, master_seed=MASTER, model=model, servers=servers, variant=variant,
                           queue_spill_cap=spill, buffers=b, diag=diag)
    out = _rows(res)
    del b
    torch.cuda.empty_cache()
    return out


_REFERENCE = {}


def reference(name):
    """Reference arrays of the shape's model and server count, from a route that never needs the general engine"""
    host_model, servers, trials, nobj, arr, srv = shape_of(name)
    key = (host_model, servers)
    if key in _REFERENCE:
        return _REFERENCE[key]
    dev = torch.device("cuda", torch.cuda.current_device())
    if host_model == 2 and servers > 14:
        ws = rings_bytes(name, trials) + 2 * estimated_need(name) + (64 << 20)
        ref = _launch(name, host_model, 0, workspace=ws)
        assert (ref["status"] == 0).all()
    else:
        diag = torch.zeros(4, dtype=torch.int64, device=dev)
        ref = _launch(name, host_model, cb.VARIANT_STATIC if host_model != 2 else 0, spill=BIG_RING, diag=diag)
        assert int(diag[2].item()) == 0 and (ref["status"] == 0).all()
    port = load_port()
    for t in range(0, trials, trials // 32):
        w = run_trials(port, "port", host_model, servers, MASTER, t, 1, nobj, arr, srv)[0]
        assert (ref["events"][t], ref["objects"][t], ref["t_end"][t], ref["sum_wait"][t]) == (w.events, w.objects, w.t_end, w.sum_wait), (name, t)
    _REFERENCE[key] = ref
    return ref


def _same(name, got, ref, rows):
    for f in FIELDS:
        g, r = got[f][rows], ref[f][rows]
        assert np.array_equal(g.view(np.uint8), r.view(np.uint8)), (name, f, np.nonzero(g != r)[0][:8])


@pytest.mark.parametrize("name", list(GPU_SHAPES))
def test_the_device_entry_flags_what_does_not_fit_and_a_larger_workspace_cures_it(name):
    ref = reference(name)
    model, variant = _model_id(name), GPU_SHAPES[name][2]
    t = time.monotonic()
    got = _launch(name, model, variant)
    flagged = got["status"] != 0
    print(f"\n{name}: default workspace, {int(flagged.sum())} of {len(flagged)} trials flagged ({time.monotonic() - t:.1f} s)")
    assert (got["status"][flagged] == cb.TRIAL_ARENA_EXHAUSTED).all(), np.unique(got["status"])
    assert flagged.any()                    # the shape exhausts the route's arena
    _same(name, got, ref, ~flagged)
    trials = shape_of(name)[2]
    ws = rings_bytes(name, trials) + 256 + estimated_need(name) * 5 // 4
    got = _launch(name, model, variant, workspace=ws)
    assert (got["status"] == 0).all(), (name, int((got["status"] != 0).sum()))
    _same(name, got, ref, slice(None))


EXP_DTYPE = np.dtype([("arr_mean", "<f8"), ("srv_mean", "<f8"), ("obj_cnt", "<u8"), ("sum_wait", "<f8"), ("events", "<u8"),
                      ("t_end", "<f8"), ("status", "<u4"), ("max_queue", "<u4"), ("counters", "<u8", (8,))])


@pytest.mark.parametrize("name", list(GPU_SHAPES))
def test_the_host_entry_reruns_what_ran_out_of_arena(name):
    ref = reference(name)
    model, variant = _model_id(name), GPU_SHAPES[name][2]
    _, servers, trials, nobj, arr, srv = shape_of(name)
    exp = np.zeros(trials, dtype=EXP_DTYPE)
    exp["arr_mean"], exp["srv_mean"] = arr, srv
    t = time.monotonic()
    cb.cimba_run_experiment(exp, model=model, num_objects=nobj, master_seed=MASTER, servers=servers, variant=variant,
                            all_gpus=name == "mm1-v0")
    print(f"\n{name}: host entry {time.monotonic() - t:.1f} s")
    assert (exp["status"] == 0).all()
    got = {"events": exp["events"], "objects": exp["obj_cnt"], "t_end": exp["t_end"], "sum_wait": exp["sum_wait"],
           "max_queue": exp["max_queue"], "counters": exp["counters"]}
    for f in FIELDS:                        # the same bits; the reference's integer columns are signed
        assert np.array_equal(np.ascontiguousarray(got[f]).view(np.uint8), np.ascontiguousarray(ref[f]).view(np.uint8)), (name, f)
