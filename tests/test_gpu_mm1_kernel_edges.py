"""Edge cases of mm1_kernel (MODEL_MM1, variant 0), the kernel bench.py measures.  It draws each variate one step ahead, and a
raw draw that needs the ziggurat slow path parks the lane until the warp's parked set, examined every 8th step, holds
MM1_COLD_BATCH lanes or every running lane.

Every test compares variant 0 bit for bit with the oracle run alone at each trial's own parameters, and with variant 1
(queue_kernel<0>, which draws each variate inside its event step), pop traces included where the case is small.  The cases:
trials that end at every step of the first three 8-step periods and in partial warps; lanes of one warp at different means
(idle ones next to ones that spill or overflow); long trials whose streams hold consecutive cold draws (counted here from the
oracle's own generator); the warp-per-trial mapping; and the TRACE instantiation."""
import math
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import cimba_b200 as cb
from oracle_libs import load_port, rng_draws, run_trials, trace_trial

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]

MASTER = 0x2545F4914F6CDD1D
FIRST = 907
WINDOW, RING = 32, 512                  # queue_model.cuh QUEUE_WINDOW, capi.cu QUEUE_SPILL_CAP
QUEUE_OVERFLOW = 1                      # CIMBA_B200_TRIAL_QUEUE_OVERFLOW
SCALES = (1.0, 0.37, 3.7, 1234.5, 0.061)
RHO = (0.9, 0.5, 1.3, 0.05, 4.0, 0.75, 0.3, 2.0, 0.99)


def _means(n, rho=RHO):
    srv = np.array([SCALES[i % len(SCALES)] for i in range(n)])
    arr = np.array([srv[i] / rho[i % len(rho)] for i in range(n)])
    return arr, srv


def _launch(arr, srv, nobj, variant, mapping=cb.MAP_LANE, trace=0):
    dev = torch.device("cuda", torch.cuda.current_device())
    a = torch.tensor(arr, dtype=torch.float64, device=dev)
    s = torch.tensor(srv, dtype=torch.float64, device=dev)
    res = cb.launch_trials(a, s, num_objects=nobj, master_seed=MASTER, first_trial=FIRST, model=cb.MODEL_MM1,
                           mapping=mapping, trace_cap=trace, variant=variant)
    torch.cuda.synchronize(dev)
    return res


def _host(res):
    """The result arrays, doubles as their bit patterns."""
    out = {k: getattr(res, k).cpu().numpy() for k in ("events", "objects", "status", "max_queue")}
    for k in ("t_end", "sum_wait"):
        out[k] = np.ascontiguousarray(getattr(res, k).cpu().numpy(), dtype=np.float64).view(np.uint64)
    if res.trace_key is not None:
        out["trace_key"] = res.trace_key.cpu().numpy()
        out["trace_time"] = np.ascontiguousarray(res.trace_time.cpu().numpy(), dtype=np.float64).view(np.uint64)
    return out


def _bits(x):
    return int(np.float64(x).view(np.uint64))


def _oracle(arr, srv, nobj):
    port = load_port()
    return [run_trials(port, "port", 0, 1, MASTER, FIRST + i, 1, nobj, float(arr[i]), float(srv[i]))[0]
            for i in range(len(arr))]


def _check_oracle(got, want, rows, tag):
    for i in rows:
        w = want[i]
        assert (int(got["events"][i]), int(got["objects"][i])) == (w.events, w.objects), (tag, i)
        assert int(got["t_end"][i]) == _bits(w.t_end) and int(got["sum_wait"][i]) == _bits(w.sum_wait), (tag, i)
        assert int(got["status"][i]) == 0, (tag, i)
        if w.max_queue <= WINDOW + RING:                # beyond the ring the repair pass re-ran the trial
            assert int(got["max_queue"][i]) == w.max_queue, (tag, i, int(got["max_queue"][i]), w.max_queue)


def _check_trace(got, arr, srv, nobj, cap, rows, tag):
    port = load_port()
    for i in rows:
        r, keys, times = trace_trial(port, "port", 0, 1, cb.fmix64(MASTER, FIRST + i), nobj, float(arr[i]), float(srv[i]), cap)
        n = len(keys)
        assert n == min(cap, r.events), (tag, i)
        assert got["trace_key"][i, :n].tolist() == keys, (tag, i)
        assert got["trace_time"][i, :n].tolist() == [_bits(t) for t in times], (tag, i)


def _check_same(v0, v1, rows, tag):
    for k in v0:
        assert np.array_equal(v0[k][rows], v1[k][rows]), (tag, k)


@pytest.mark.parametrize("nobj", range(1, 25))
def test_every_step_position(nobj):
    """num_objects 1..24 ends trials at every step of the first three 8-step periods; 37 + nobj trials leave a partial warp (and, from
    28 objects of trials on, a partial CTA).  Full pop traces against the oracle and variant 1."""
    n = 37 + nobj
    arr, srv = _means(n)
    cap = 4 * nobj + 8
    want = _oracle(arr, srv, nobj)
    assert max(w.events for w in want) <= cap
    v0, v1 = _host(_launch(arr, srv, nobj, 0, trace=cap)), _host(_launch(arr, srv, nobj, 1, trace=cap))
    rows = list(range(n))
    _check_oracle(v0, want, rows, "variant 0")
    _check_trace(v0, arr, srv, nobj, cap, rows, "variant 0")
    _check_same(v0, v1, rows, "variant 0 vs 1")


def test_mixed_means_within_a_warp():
    """Lanes of one warp at rho from 0.05 (mostly idle) to 4 (past the on-chip window, the spill ring and its end): the parked
    set and the look-ahead draw must stay per lane.  Trials that overflow the ring are re-run by the repair pass; variant 1 has none,
    so the two variants are compared on the other trials."""
    n, nobj, cap = 197, 3000, 2000
    arr, srv = _means(n)
    want = _oracle(arr, srv, nobj)
    v0, v1 = _host(_launch(arr, srv, nobj, 0, trace=cap)), _host(_launch(arr, srv, nobj, 1, trace=cap))
    assert any(WINDOW < w.max_queue <= WINDOW + RING for w in want)          # spilled, within the ring
    assert any(w.max_queue > WINDOW + RING for w in want)                    # overflowed
    assert any(w.max_queue <= 2 for w in want)                              # idle
    _check_oracle(v0, want, range(n), "variant 0")
    on_chip = [i for i in range(n) if want[i].max_queue <= WINDOW + RING]    # ran to the end in mm1_kernel
    _check_trace(v0, arr, srv, nobj, cap, on_chip, "variant 0")
    clean = [i for i in range(n) if int(v1["status"][i]) == 0]
    assert len(clean) < n and [i for i in range(n) if int(v1["status"][i]) & QUEUE_OVERFLOW]
    _check_same(v0, v1, clean, "variant 0 vs 1")


def _zig_exp_tables():
    """The exponential ziggurat's tables, from the oracle's generated header."""
    txt = (ROOT / "oracle/port/zig_tables.h").read_text()

    def table(name, conv):
        body = re.search(r"zt_exp_%s\[256\] = \{(.*?)\};" % name, txt, re.S).group(1)
        vals = [conv(v.strip()) for v in body.replace("\n", " ").split(",") if v.strip()]
        assert len(vals) == 256, name
        return vals

    hexu = lambda s: int(s.rstrip("ULul"), 16)      # noqa: E731
    t = {"x": table("x", float), "y": table("y", float), "concavity": table("concavity", hexu), "prob": table("prob", hexu),
         "alias": table("alias", int)}
    t["max"] = int(re.search(r"#define ZT_EXP_MAX (\d+)u", txt).group(1))
    t["tail"] = float(re.search(r"#define ZT_EXP_TAIL (\S+)", txt).group(1))
    return t


def _cold_flags(seed, n):
    """Which of a stream's first n standard exponentials took the ziggurat slow path.  The walk restates the oracle's
    std_exponential over its raw sfc64 draws and must reproduce the oracle's own exponentials bit for bit."""
    t = _zig_exp_tables()
    m = n + n // 4 + 64
    raw = [int(v) for v in rng_draws(load_port(), "port", seed, 0, 0.0, 0.0, m).view(np.uint64)]
    top = (1 << 64) - 1
    pos = 0

    def nxt():
        nonlocal pos
        pos += 1
        return raw[pos - 1]

    def slow(ux):
        shift = 0.0
        while True:
            uy = nxt()
            j = uy & 0xff
            if nxt() >= t["prob"][j]:
                j = t["alias"][j]
            if j > 0:
                while True:
                    if uy > top - ux:
                        uy, ux = top - uy, top - ux
                    gap = (top - ux) - uy
                    x = math.ldexp(t["x"][j], 64) + (t["x"][j - 1] - t["x"][j]) * float(ux)
                    if gap >= t["concavity"][j]:
                        return x + shift
                    y = math.ldexp(t["y"][j - 1], 64) + (t["y"][j] - t["y"][j - 1]) * float(uy)
                    if y <= math.exp(-x):
                        return x + shift
                    uy, ux = nxt(), nxt()
            shift += t["tail"]
            ux = nxt()
            if (ux & 0xff) <= t["max"]:
                return t["x"][ux & 0xff] * float(ux) + shift

    vals, cold = [], []
    for _ in range(n):
        u = nxt()
        hot = (u & 0xff) <= t["max"]
        vals.append(t["x"][u & 0xff] * float(u) if hot else slow(u))
        cold.append(not hot)
    assert pos <= m
    want = rng_draws(load_port(), "port", seed, 1, 1.0, 0.0, n)
    assert np.array_equal(np.array(vals).view(np.uint64), want.view(np.uint64))
    return cold


def test_long_trials_with_consecutive_cold_draws():
    """10^5 objects per trial: every trial's stream has runs of consecutive cold draws, so a lane parks again right after its
    slow path ran."""
    n, nobj = 45, 100_000
    arr, srv = _means(n, rho=(0.9, 0.5, 0.99, 0.3, 0.8))
    runs = 0
    for i in (0, 1, 2):
        cold = _cold_flags(cb.fmix64(MASTER, FIRST + i), nobj)      # a trial draws at least nobj variates
        runs += sum(1 for k in range(1, nobj) if cold[k] and cold[k - 1])
    assert runs >= 1
    want = _oracle(arr, srv, nobj)
    v0, v1 = _host(_launch(arr, srv, nobj, 0)), _host(_launch(arr, srv, nobj, 1))
    _check_oracle(v0, want, range(n), "variant 0")
    _check_same(v0, v1, list(range(n)), "variant 0 vs 1")


def test_warp_per_trial_mapping():
    """mapping 32: lane 0 of each warp simulates and the other 31 lanes must neither draw nor park."""
    n, nobj, cap = 45, 700, 3000
    arr, srv = _means(n)
    want = _oracle(arr, srv, nobj)
    v0 = _host(_launch(arr, srv, nobj, 0, mapping=cb.MAP_WARP, trace=cap))
    v1 = _host(_launch(arr, srv, nobj, 1, mapping=cb.MAP_WARP, trace=cap))
    lane = _host(_launch(arr, srv, nobj, 0))
    _check_oracle(v0, want, range(n), "variant 0, mapping 32")
    _check_trace(v0, arr, srv, nobj, cap, [i for i in range(n) if want[i].max_queue <= WINDOW + RING], "variant 0, mapping 32")
    clean = [i for i in range(n) if int(v1["status"][i]) == 0]
    _check_same(v0, v1, clean, "variant 0 vs 1, mapping 32")
    for k in lane:
        assert np.array_equal(v0[k], lane[k]), k


def test_trace_instantiation_matches_plain():
    """The TRACE instantiation computes what the plain one does, and its pops are the oracle's."""
    n, nobj, cap = 100, 400, 1700
    arr, srv = _means(n)
    traced, plain = _host(_launch(arr, srv, nobj, 0, trace=cap)), _host(_launch(arr, srv, nobj, 0))
    for k in plain:
        assert np.array_equal(traced[k], plain[k]), k
    want = _oracle(arr, srv, nobj)
    _check_oracle(plain, want, range(n), "plain")
    _check_trace(traced, arr, srv, nobj, cap, range(n), "traced")
