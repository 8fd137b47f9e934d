"""GPU parity when every trial carries its own parameters (tests/param_cases.py): every launch path of every model, the repair
passes with flagged and clean trials interleaved, the host-buffer entry with an unusual struct layout, and the on-device folds
of per-trial results at sizes that leave some of their 256 partial sums empty.

Each trial is compared bit for bit with the oracle run alone at that trial's own (arr_mean, srv_mean) and seed: a kernel that
reads another trial's parameters (the first of its warp, CTA or persistent run), or drops the service mean's multiply on a rare
path, fails here.  Each test also asserts the precondition that makes it bite (queues in the window, the ring and beyond it;
harbors with more ships than the on-chip tables hold; different means within one persistent warp), so that a change of the table
cannot quietly weaken it."""
import ctypes as C
import functools
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from oracle_libs import load_port, load_ref
from param_cases import FIRST, MASTER, N, RHO, RHO_REPAIR, TABLE, TRACE_POPS, oracle, oracle_trace, per_trial_params

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]

WINDOW, RING = 32, 512              # queue_model.cuh QUEUE_WINDOW / pool_model.cuh POOL_WINDOW, capi.cu QUEUE_SPILL_CAP
HARBOR_ON_CHIP, HARBOR_HBM = 43, 120  # ships alive the warp-per-trial tables / the lane-per-trial tables hold
QUEUE_OVERFLOW = 1                  # CIMBA_B200_TRIAL_QUEUE_OVERFLOW
TRACED = (0, 3, 6, 40, N - 1)       # trial 3: rho 1.3 (spill ring), 6 and 40: rho 4 (beyond the ring)
GEN, STA = cb.VARIANT_GENERAL, cb.VARIANT_STATIC
BUILTIN = {0: cb.MODEL_MM1, 1: cb.MODEL_GG1, 2: cb.MODEL_MMC, 3: cb.MODEL_GUARDED, 4: cb.MODEL_PREEMPT, 5: cb.MODEL_BUFFER,
           6: cb.MODEL_PRIOQ, 7: cb.MODEL_HOLD, 8: cb.MODEL_TIMERS, 9: cb.MODEL_MM1_RECORDED, 10: cb.MODEL_HARBOR,
           11: cb.MODEL_GUARDED_RECORDED, 12: cb.MODEL_BUFFER_RECORDED, 13: cb.MODEL_PRIOQ_RECORDED,
           14: cb.MODEL_RESOURCE_RECORDED, 16: cb.MODEL_RENEGE, 19: cb.MODEL_TUTORIAL1}
REF_ONLY = (16, 17, 19)             # models of the reference driver only: checked against the live reference build
ALL8 = (3, 4, 5, 6, 8, 9, 10, 11, 12, 13, 14, 19)   # all eight counters are the reference's (cmb_engine_vectors.json "all8")


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _counts(t):
    return np.ascontiguousarray(t.cpu().numpy(), dtype=np.int64).view(np.uint64)


def _ref():
    ref = load_ref()
    if ref is None:
        pytest.skip("oracle/_ref/librefdrv.so did not travel with this snapshot")
    ref.ref_set_param.argtypes = [C.c_int, C.c_double]
    return ref


def _checker(model):
    return (_ref(), "ref") if model in REF_ONLY else (load_port(), "port")


@functools.lru_cache(maxsize=None)
def _want(model, servers, rho=RHO):
    """(arr, srv, oracle results) of the table's N trials."""
    nobj, params = TABLE[model][1], TABLE[model][3]
    arr, srv = per_trial_params(model, servers=servers, rho=rho)
    lib, prefix = _checker(model)
    if params:
        lib.ref_set_param(0, params[0])
    try:
        want = oracle(lib, prefix, model, servers, nobj, arr, srv, par=1 if model == 16 else 0)
    finally:
        if params:
            lib.ref_set_param(0, 0.0)
    return arr, srv, want


def _trace_want(model, servers, arr, srv, i):
    lib, prefix = _checker(model)
    params = TABLE[model][3]
    if params:
        lib.ref_set_param(0, params[0])
    try:
        return oracle_trace(lib, prefix, model, servers, TABLE[model][1], arr, srv, i, cb.fmix64)
    finally:
        if params:
            lib.ref_set_param(0, 0.0)


@functools.lru_cache(maxsize=None)
def _user_model(stem):
    so = ROOT / "cimba_b200/lib/models" / f"lib{stem}.so"
    if not so.exists():                                 # built by __graft_entry__.build(); nvcc is on the GPU machine too
        sys.path.insert(0, str(ROOT / "scripts"))
        import build_model
        build_model.build(ROOT / "examples" / f"{stem}.cu")
    return cb.load_model(so)


def _launch(model_id, servers, nobj, arr, srv, variant=0, mapping=0, spill=0, trace=0, params=(), first=FIRST):
    dev = torch.device("cuda", torch.cuda.current_device())
    a = torch.tensor(arr, dtype=torch.float64, device=dev)
    s = torch.tensor(srv, dtype=torch.float64, device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(a, s, num_objects=nobj, master_seed=MASTER, first_trial=first, model=model_id, servers=servers,
                           mapping=mapping, trace_cap=trace, variant=variant, queue_spill_cap=spill, params=params, diag=diag)
    torch.cuda.synchronize(dev)
    return res, [int(v) for v in diag.cpu().tolist()]


def _beyond(spill):
    return WINDOW + (spill or RING)


def _expected_max_queue(model, variant, spill, w):
    """What max_queue holds on this path, or None where the path does not report it (the general engine's M/M/1 and G/G/1
    write 0, its hold model the list's capacity)."""
    if model in (0, 1):
        return w.max_queue if variant in (0, 1, 2) and w.max_queue <= _beyond(spill) else None
    if model in (2, 10, 11, 12, 13, 14):
        return w.max_queue
    if model in (3, 4, 5, 6, 8) or (model == 7 and variant != GEN):
        return w.max_fel
    return None


def _compare(res, want, model, variant=0, spill=0, rows=None, tag=""):
    ev, ob, st = _counts(res.events), _counts(res.objects), res.status.cpu().numpy()
    te, sw, mq = _u64(res.t_end.cpu().numpy()), _u64(res.sum_wait.cpu().numpy()), res.max_queue.cpu().numpy()
    cnt = _counts(res.counters)
    ncnt = 8 if model in ALL8 and not (model == 7 and variant == GEN) else (4 if model in (7, 16, 17) else 0)
    for i in (range(len(want)) if rows is None else rows):
        w = want[i]
        got = (int(ev[i]), int(ob[i]), int(te[i]), int(sw[i]), int(st[i]))
        exp = (w.events, w.objects, int(_u64([w.t_end])[0]), int(_u64([w.sum_wait])[0]), 0)
        assert got == exp, (tag, i, got, exp)
        if ncnt:
            assert [int(v) for v in cnt[i][:ncnt]] == w.counters()[:ncnt], (tag, i, "counters")
        m = _expected_max_queue(model, variant, spill, w)
        if m is not None:
            assert int(mq[i]) == m, (tag, i, "max_queue", int(mq[i]), m)


def _assert_coverage(model, servers, arr, want, variant):
    mq = np.array([w.max_queue for w in want])
    if model == 0:          # the window, the HBM spill ring and beyond it, in one launch
        assert (mq <= WINDOW).any() and ((mq > WINDOW) & (mq <= WINDOW + RING)).any() and (mq > WINDOW + RING).any(), mq
    if model == 10:         # more ships alive than the warp-per-trial tables hold, and fewer, never more than the HBM tables
        assert mq.min() < HARBOR_ON_CHIP < mq.max() < HARBOR_HBM, (mq.min(), mq.max())
    if model == 7:          # the hold kernels put 1, 2 or 4 consecutive trials on one warp: their means differ
        assert all(len(set(arr[k:k + 4].tolist())) == len(arr[k:k + 4]) for k in range(0, len(arr), 4))
    # every warp of trials mixes parameter values
    assert all(len(set(arr[k:k + 32].tolist())) > 1 for k in range(0, len(arr) - 1, 32))


# (model, servers, variant, mapping, queue_spill_cap, library): every launch path cimba_b200_launch accepts for the model
PATHS = ([(0, 1, v, m, 0, None) for v in (0, 1) for m in (1, 32)] + [(0, 1, 2, 1, 0, None), (0, 1, STA, 1, 0, None),
                                                                     (0, 1, GEN, 1, 0, None), (0, 1, 0, 1, 4096, None)]
         + [(1, 1, v, 1, 0, None) for v in (0, 1, STA, GEN)]
         + [(2, c, v, 1, 0, None) for c in (3, 8) for v in (0, 1, GEN)]
         + [(9, 1, v, 1, 0, None) for v in (0, STA, GEN)]
         + [(7, 300, v, 1, 0, None) for v in (0, 1, 2, 3, 4, GEN)]
         + [(10, 6, v, 1, 0, None) for v in (0, 2, GEN)]
         + [(m, TABLE[m][0], v, 1, 0, None) for m in (3, 4, 5, 6, 8, 11, 12, 13, 14) for v in (0, GEN)]
         + [(16, 40, 0, 1, 0, None), (19, 1, 0, 1, 0, None), (19, 1, GEN, 1, 0, None)]
         + [(0, 1, 0, 1, 0, "mm1_user_model"), (0, 1, 0, 1, 0, "mm1_static_user_model"),
            (17, 4, 0, 1, 0, "tandem_user_model"), (17, 4, 0, 1, 0, "tandem_static_user_model")])


def _path_id(p):
    model, servers, variant, mapping, spill, lib = p
    v = {GEN: "general", STA: "static"}.get(variant, f"v{variant}")
    return f"model{model}-s{servers}-{v}" + ("-warp" if mapping == 32 else "") + (f"-spill{spill}" if spill else "") + \
        (f"-{lib}" if lib else "")


@pytest.mark.parametrize("path", PATHS, ids=_path_id)
def test_every_trial_matches_the_oracle_at_its_own_parameters(path):
    model, servers, variant, mapping, spill, lib = path
    arr, srv, want = _want(model, servers)
    _assert_coverage(model, servers, arr, want, variant)
    model_id = _user_model(lib) if lib else BUILTIN[model]
    nobj, params = TABLE[model][1], TABLE[model][3]
    tag = _path_id(path)
    for trace in (0, TRACE_POPS):
        res, _ = _launch(model_id, servers, nobj, arr, srv, variant, mapping, spill, trace, params)
        flagged = [i for i, w in enumerate(want) if model in (0, 1) and variant == 1 and w.max_queue > _beyond(spill)]
        if flagged:         # variant 1 of M/M/1 and G/G/1 has no repair pass: overflowed trials are flagged, the others exact
            st = res.status.cpu().numpy()
            assert [i for i in range(N) if st[i] & QUEUE_OVERFLOW] == flagged, tag
        rows = [i for i in range(N) if i not in flagged]
        _compare(res, want, model, GEN if lib else variant, spill, rows, tag)    # the libraries run the authoring surface
        if trace:
            keys, times = res.trace_key.cpu().numpy(), res.trace_time.cpu().numpy()
            for i in (i for i in TRACED if i not in flagged):
                r, k, t = _trace_want(model, servers, arr, srv, i)
                m = min(TRACE_POPS, r.events)
                assert list(keys[i, :m]) == k, (tag, i)
                assert np.array_equal(_u64(times[i, :m]), _u64(np.array(t))), (tag, i)


def test_harbor_warp_per_trial_only_is_exact_where_it_reports_success():
    """variant 1 runs every trial warp-per-trial with its state in shared memory and flags what outgrows those tables."""
    arr, srv, want = _want(10, 6)
    _assert_coverage(10, 6, arr, want, 1)
    res, _ = _launch(cb.MODEL_HARBOR, 6, TABLE[10][1], arr, srv, variant=1)
    ok = [i for i, s in enumerate(res.status.cpu().tolist()) if s == 0]
    assert len(ok) > N // 2
    assert any(want[i].max_queue > 30 for i in ok)
    _compare(res, want, 10, 1, rows=ok, tag="harbor v1")


@pytest.mark.parametrize("variant", [0, 1])
def test_hold_persistent_warps_run_trials_with_different_means(variant):
    """More trials than any H100 keeps resident (SMs x 64 warps), every trial with a mean of its own: the persistent warps of
    hold_deep_kernel (variant 0) and hold_kernel (variant 1) loop, and every later trial of a warp must use its own mean."""
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    n = props.multi_processor_count * getattr(props, "max_threads_per_multi_processor", 2048) // 32 + 101
    workers, dur = 300, 3
    cyc = (0.5, 0.93, 2.0, 0.7, 1.3, 0.61, 1.7)
    arr = np.array([cyc[i % 7] * (1.0 + i / (4.0 * n)) for i in range(n)])
    srv = np.full(n, 0.37)
    assert len(set(arr.tolist())) == n                  # so any two trials one warp runs differ in their mean
    res, _ = _launch(cb.MODEL_HOLD, workers, dur, arr, srv, variant=variant, first=0)
    ev, sw, st = _counts(res.events), _u64(res.sum_wait.cpu().numpy()), res.status.cpu().numpy()
    port = load_port()
    for i in sorted(set(range(0, n, 13)) | set(range(n - 128, n))):
        r, _, _ = oracle_trace(port, "port", 7, workers, dur, arr, srv, i, cb.fmix64, first=0, cap=0)
        assert (int(ev[i]), int(sw[i]), int(st[i])) == (r.events, int(_u64([r.sum_wait])[0]), 0), (variant, i)


# ------------------------------------------------------------------ repair passes with flagged trials interleaved

@pytest.mark.parametrize("model,servers,variant", [(0, 1, 0), (0, 1, 2), (0, 1, STA), (0, 1, 1), (1, 1, 0), (2, 3, 0),
                                                   (2, 8, 0), (2, 8, 1), (9, 1, 0)])
def test_repair_pass_reruns_exactly_the_flagged_trials(model, servers, variant):
    """rho = 4 on every 7th trial, rho <= 0.9 on the others, time scales from 1e-3 to 1234.5: the fast kernel flags the trials
    whose queue (M/M/c: wait list) outgrows window + ring (`put_far` and its overflow branch in mm1_fast.cuh, mm1_pc.cuh,
    gg1_fast.cuh, queue_model.cuh, pool_fast.cuh, the StampRing of cmb_static.cuh), and the repair pass re-runs those and no
    other on the general engine at their own parameters.  diag[2] counts the re-run trials."""
    arr, srv, want = _want(model, servers, RHO_REPAIR)
    mq = np.array([w.max_queue for w in want])
    # M/M/c's max_queue counts customers alive (waiting + in service): no trial may sit where that count is ambiguous
    margin = servers + 2 if model == 2 else 0
    assert not ((mq > WINDOW + RING - margin) & (mq <= WINDOW + RING + margin)).any()
    over = [i for i in range(N) if mq[i] > WINDOW + RING + margin]
    assert over == [i for i in range(N) if i % 7 == 6]  # interleaved: every warp has flagged and clean trials
    res, diag = _launch(BUILTIN[model], servers, TABLE[model][1], arr, srv, variant)
    if variant == 1 and model == 0:                     # no repair pass: the flag is the answer
        st = res.status.cpu().numpy()
        assert [i for i in range(N) if st[i] & QUEUE_OVERFLOW] == over
        _compare(res, want, model, variant, rows=[i for i in range(N) if i not in over], tag="flagged")
        return
    _compare(res, want, model, variant, tag=(model, servers, variant))
    assert diag[2] == len(over), (diag, len(over))


# ------------------------------------------------------------------ the host-buffer entry with per-trial parameters

# srv_mean before arr_mean, a 4-byte field first (no field 8-aligned), an odd stride
HB_DTYPE = np.dtype({"names": ["tag", "srv_mean", "arr_mean", "obj_cnt", "sum_wait", "events", "t_end", "status", "max_queue",
                               "counters"],
                     "formats": ["<u4", "<f8", "<f8", "<u8", "<f8", "<u8", "<f8", "<u4", "<u4", ("<u8", (8,))],
                     "offsets": [0, 4, 12, 20, 28, 36, 44, 52, 56, 60], "itemsize": 125})


@pytest.mark.parametrize("model,servers", [(0, 1), (2, 3), (10, 6)])
def test_host_buffer_entry_with_per_trial_parameters(model, servers, monkeypatch):
    arr, srv, want = _want(model, servers)
    nobj = TABLE[model][1]
    exp = np.zeros(N, dtype=HB_DTYPE)
    exp["tag"] = 0xA5A50000 + np.arange(N)
    exp["arr_mean"], exp["srv_mean"] = arr, srv
    chunked, sharded = exp.copy(), exp.copy()
    run = dict(model=BUILTIN[model], num_objects=nobj, master_seed=MASTER, first_trial=FIRST, servers=servers)
    cb.cimba_run_experiment(exp, **run)
    cb.cimba_run_experiment(sharded, all_gpus=True, **run)
    monkeypatch.setenv("CIMBA_B200_CHUNK_TRIALS", "97")
    cb.cimba_run_experiment(chunked, **run)
    for f in HB_DTYPE.names:
        assert np.array_equal(exp[f], chunked[f]) and np.array_equal(exp[f], sharded[f]), f
    assert (exp["tag"] == 0xA5A50000 + np.arange(N)).all() and (exp["arr_mean"] == arr).all() and (exp["srv_mean"] == srv).all()
    for i, w in enumerate(want):
        row = exp[i]
        assert (int(row["events"]), int(row["obj_cnt"]), int(row["status"])) == (w.events, w.objects, 0), i
        assert float(row["t_end"]).hex() == w.t_end.hex() and float(row["sum_wait"]).hex() == w.sum_wait.hex(), i
        m = _expected_max_queue(model, 0, 0, w)
        if m is not None:
            assert int(row["max_queue"]) == m, i
        if model == 10:
            assert [int(v) for v in row["counters"]] == w.counters(), i
    if model != 10:         # M/M/1 and M/M/c write no counters: zeros, not what an earlier call left in the reused arena
        assert not exp["counters"].any()


# ------------------------------------------------------------------ the device folds at sizes that leave partial sums empty

def _tree(items, empty, add, merge, block=256):
    """summary.cuh's order: thread t folds items t, t + 256, ... then a halving tree 128 -> 1."""
    part = []
    for t in range(block):
        acc = empty()
        for i in range(t, len(items), block):
            acc = add(acc, items[i])
        part.append(acc)
    k = block // 2
    while k > 0:
        for i in range(k):
            part[i] = merge(part[i], part[i + k])
        k //= 2
    return part[0]


def _data_add(acc, y):
    acc.add(y)
    return acc


def _wtd_add(acc, xw):
    acc.add(*xw)
    return acc


def _close(a, b):
    # tree and serial fold differ by the order of Pebay's updates only: each update rounds the moments to a few ulp, and with
    # n <= 4097 samples over at most 17 tree levels plus 16 serial adds per thread the difference stays far below 1e-9 relative
    # (the BASELINE.json tolerance); moments of fewer than three samples are undefined (NaN / 0) in both
    return (math.isnan(a) and math.isnan(b)) or abs(a - b) <= 1e-9 * max(abs(a), abs(b), 1e-300)


@functools.lru_cache(maxsize=None)
def _averages():
    """4097 per-trial average times in system of an M/M/1 launch at the table's parameters: 1e-3 .. 1e4."""
    arr, srv = per_trial_params(0, n=4097, rho=RHO_REPAIR)
    res, _ = _launch(cb.MODEL_MM1, 1, 200, arr, srv)
    assert res.status.abs().sum().item() == 0
    return res.sum_wait.clone(), res.objects.clone()


@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 1000, 4097])
def test_device_summary_is_the_host_tree_bit_for_bit(n):
    sw, ob = _averages()
    sw, ob = sw[:n].contiguous(), ob[:n].contiguous()
    dev = cb.summarize_on_device(sw, ob).cpu().tolist()
    avg = (sw.cpu().numpy() / ob.cpu().numpy().astype(np.float64)).tolist()
    if n >= 255:
        assert max(avg) / min(avg) > 1e5               # averages spanning orders of magnitude
    host = _tree(avg, cb.DataSummary, _data_add, cb.DataSummary.merge)
    assert _u64(dev[:7]).tolist() == _u64(host.to_list()[:7]).tolist(), n
    serial = cb.DataSummary.of(avg)
    d = cb.DataSummary.from_list(dev)
    assert d.count() == serial.count() == n and d.min() == serial.min() and d.max() == serial.max()
    for a, b in ((d.mean(), serial.mean()), (d.variance(), serial.variance()), (d.skewness(), serial.skewness()),
                 (d.kurtosis(), serial.kurtosis())):
        assert _close(a, b), (n, a, b)


@pytest.mark.parametrize("n", [1, 2, 100, 255, 256, 257, 1000, 4097])
def test_device_weighted_summary_with_zero_weights_is_the_host_tree(n):
    """Every 5th weight is zero (threads 0, 5, 10, ... start with one): cmb_wtdsummary_add skips those samples."""
    sw, ob = _averages()
    x = (sw[:n] / ob[:n].double()).contiguous()
    w = torch.tensor([0.0 if i % 5 == 0 else (0.37, 3.7, 1234.5, 0.061)[i % 4] for i in range(n)], dtype=torch.float64,
                     device=x.device)
    dev = [int(v) & (2**64 - 1) for v in cb.summarize_weighted_on_device(x, w).cpu().tolist()]
    pairs = list(zip(x.cpu().tolist(), w.cpu().tolist()))
    host = _tree(pairs, cb.WtdSummary, _wtd_add, cb.WtdSummary.merge)
    assert dev == host.to_row(), n
    serial = cb.WtdSummary()
    for p in pairs:
        serial.add(*p)
    d = cb.WtdSummary.from_row(dev)
    assert d.count() == serial.count() == sum(1 for _, v in pairs if v != 0.0)
    for a, b in ((d.mean(), serial.mean()), (d.variance(), serial.variance()), (d.skewness(), serial.skewness()),
                 (d.kurtosis(), serial.kurtosis()), (d.wsum(), serial.wsum())):
        assert _close(a, b), (n, a, b)


@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 1000])
def test_device_row_merge_with_empty_rows_is_the_host_tree(n):
    """Per-trial rows of recorded M/M/1 trials at their own parameters, every 3rd row empty (count 0), row 0 included."""
    arr, srv = per_trial_params(9, n=n, rho=RHO_REPAIR)
    res, _ = _launch(cb.MODEL_MM1_RECORDED, 1, 300, arr, srv)
    rows = res.counters.clone()
    empty = torch.from_numpy(np.array(cb.WtdSummary().to_row(), dtype=np.uint64).view(np.int64)).to(rows.device)
    rows[0::3] = empty
    dev = [int(v) & (2**64 - 1) for v in cb.merge_weighted_rows_on_device(rows).cpu().tolist()]
    host_rows = [cb.WtdSummary.from_row(r) for r in _counts(rows).tolist()]
    assert all(r.count() == 0 for r in host_rows[0::3]) and all(r.count() > 0 for r in host_rows[1::3])
    host = _tree(host_rows, cb.WtdSummary, cb.WtdSummary.merge, cb.WtdSummary.merge)
    assert dev == host.to_row(), n
    serial = cb.WtdSummary()
    for r in host_rows:
        serial = cb.WtdSummary.merge(serial, r)
    d = cb.WtdSummary.from_row(dev)
    assert d.count() == serial.count()
    for a, b in ((d.mean(), serial.mean()), (d.variance(), serial.variance()), (d.wsum(), serial.wsum())):
        assert _close(a, b), (n, a, b)


def test_device_folds_refuse_an_empty_input():
    """include/cimba_b200.h: n = 0 returns CIMBA_B200_EINVAL and leaves the output untouched."""
    dev = torch.device("cuda", torch.cuda.current_device())
    x = torch.ones(4, dtype=torch.float64, device=dev)
    o = torch.ones(4, dtype=torch.int64, device=dev)
    out = torch.full((8,), 7.0, dtype=torch.float64, device=dev)
    row = torch.full((8,), 7, dtype=torch.int64, device=dev)
    rows = torch.zeros((4, 8), dtype=torch.int64, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert cb.lib.cimba_b200_summarize(x.data_ptr(), o.data_ptr(), 0, out.data_ptr(), stream) == -1
    assert cb.lib.cimba_b200_summarize_weighted(x.data_ptr(), x.data_ptr(), 0, row.data_ptr(), stream) == -1
    assert cb.lib.cimba_b200_merge_weighted_rows(rows.data_ptr(), 0, row.data_ptr(), stream) == -1
    torch.cuda.synchronize(dev)
    assert (out == 7.0).all() and (row == 7).all()
    with pytest.raises(cb.CimbaError):
        cb.summarize_on_device(x[:0], o[:0])
