"""GPU side of the cmb_random parameter sweep (tests/random_sweep_cases.py): every case drawn on the device by
cimba_b200_rng_draws_ex (rng_draws_ex_kernel, the general path's formulation), N variates at the case's seed.  Each case was
first shown to finish within its work bound on the host build (tests/test_random_sweep.py).

  * kinds whose variate is no libm result: bit for bit the reference's stream - the SHA-256 in
    tests/golden/random_sweep_vectors.json, and the live reference build where it was built (a NaN as a NaN);
  * the gamma family (the Marsaglia-Tsang loop compares a log() with another expression, and CUDA's log is not glibc's): the
    same, for every case whose smallest comparison margin on the host build exceeds MARGIN_ULP; the others only finish;
  * logistic, weibull, pareto, gamma and chisquared with shape < 1: each variate recomputed in mpmath from the uniform or
    exponential it came from (drawn again on the device by the bit-exact kinds 3 / 1, or for gamma the two factors of the
    host build), the libm call correctly rounded and then moved by up to LIBM_ULP in either direction - the device value must
    lie inside that bracket.  F and t with a pow() inside: within 16 eps of the host build's value;
  * geometric, negative binomial and pascal: every variate the reference's, recomputed from the device's exponentials with
    glibc's log and gcc's conversion (modulo 2^32 past 2^32); a quotient within 4 ulp of an integer (mpmath) may differ;
  * the sweep as model code (tests/random_sweep_model.cuh, built here with scripts/build_model.py and loaded with
    cimba_b200_model_load) on the general engine and on the static tier, one trial per case: both give the counters of the
    path-1 device stream bit for bit, libm kinds included, status 0, no trial handed on by the static library (diag[2]), and
    a clock after the sampled holds equal to their sum.
Every launch first checks that the host build finished its case within the case's work bound (the golden file's call count)."""
import json
import math
import sys

import mpmath
import numpy as np
import pytest
import torch

import random_sweep_cases as rc
from oracle_libs import rng_draws_ex

pytestmark = pytest.mark.gpu

GOLD = {c["id"]: c for c in json.loads((rc.ROOT / "tests/golden/random_sweep_vectors.json").read_text())["cases"]}
MARGIN_ULP = 16.0
LIBM_ULP = 2
mpmath.mp.prec = 120


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return rc.build_host(tmp_path_factory.mktemp("random_sweep_gpu"))


def proven(i):
    """The host build drew case i within its work bound (tests/test_random_sweep.py checks the recorded count is fresh)."""
    kind, par = rc.CASES[i]
    calls = GOLD[rc.IDS[i]]["calls"]
    assert calls <= rc.N * rc.calls_bound(kind, par), (rc.IDS[i], calls)


def device(cb, i, n=rc.N):
    proven(i)
    k, p = rc.CASES[i]
    return cb.rng_draws_ex(rc.case_seed(i), k, n, p).cpu().numpy()


def exact_ok(i):
    kind, par = rc.CASES[i]
    g = GOLD[rc.IDS[i]]
    return kind not in rc.GAMMA_FAMILY or (g["margin"] is None or g["margin"] > MARGIN_ULP)


def mp_pow(b, r):
    """b^r in mpmath, b >= 0 and r > 0; 0 or inf straight away where the double result cannot be anything else."""
    if b == 0.0 or b == 1.0:
        return mpmath.mpf(b)
    lg = r * math.log2(b)
    if lg < -1200.0:
        return mpmath.mpf(0)
    if lg > 1100.0:
        return mpmath.inf
    return mpmath.mpf(b) ** mpmath.mpf(r)


def bracket(y_mp, post):
    """post(y) for the double y0 nearest y_mp and for y0 moved LIBM_ULP places down and up: (lo, hi) of the results."""
    y0 = np.array([float(y) for y in y_mp])
    down, up = y0.copy(), y0.copy()
    for _ in range(LIBM_ULP):
        down, up = np.nextafter(down, -np.inf), np.nextafter(up, np.inf)
    with np.errstate(all="ignore"):
        a, b = post(down), post(up)
    return np.minimum(a, b), np.maximum(a, b)


def assert_inside(dev, lo, hi, what):
    same = (dev == lo) | (dev == hi) | ((dev >= lo) & (dev <= hi))
    bad = np.flatnonzero(~same)
    assert bad.size == 0, (what, bad[:5], dev[bad[:3]], lo[bad[:3]], hi[bad[:3]])


BIT_EXACT = [i for i, (k, p) in enumerate(rc.CASES) if not rc.libm_value(k, p) and k not in rc.GEOMETRIC_KINDS]
LIBM_DIRECT = [i for i, (k, p) in enumerate(rc.CASES) if k in (11, 18, 19) or (k in (15, 20) and rc.libm_value(k, p))]
LIBM_COMPOSITE = [i for i, (k, p) in enumerate(rc.CASES) if k in (21, 22) and rc.libm_value(k, p)]
GEOMETRIC = [i for i, (k, _) in enumerate(rc.CASES) if k in rc.GEOMETRIC_KINDS]


@pytest.mark.parametrize("i", BIT_EXACT, ids=[rc.IDS[i] for i in BIT_EXACT])
def test_device_stream_is_the_reference_stream(cb, ref, i):
    kind, par = rc.CASES[i]
    if not exact_ok(i):
        pytest.skip(f"a log comparison within {MARGIN_ULP} ulp of a tie on the host build")
    dev = device(cb, i)
    assert rc.stream_sha256(rc.canonical(dev)) == GOLD[rc.IDS[i]]["sha256"]
    if ref is not None:
        want = rc.canonical(np.array(rng_draws_ex(ref, "ref", rc.case_seed(i), kind, par, rc.N)))
        bad = np.flatnonzero(rc.canonical(dev).view(np.uint64) != want.view(np.uint64))
        assert bad.size == 0, (bad[:5], dev[bad[:3]], want[bad[:3]])


def test_most_gamma_family_cases_demand_bit_exactness():
    fam = [i for i, (k, p) in enumerate(rc.CASES) if k in rc.GAMMA_FAMILY]
    assert sum(exact_ok(i) for i in fam) >= 0.9 * len(fam)


@pytest.mark.parametrize("i", LIBM_DIRECT, ids=[rc.IDS[i] for i in LIBM_DIRECT])
def test_libm_variates_within_two_ulp_of_the_correctly_rounded_libm_call(cb, host, i):
    kind, par = rc.CASES[i]
    if not exact_ok(i):
        pytest.skip(f"a log comparison within {MARGIN_ULP} ulp of a tie on the host build")
    dev = device(cb, i)
    seed = rc.case_seed(i)
    mp = mpmath.mpf
    if kind == 11:                                          # m + s * log(x / (1 - x))
        x = cb.rng_draws(seed, 3, rc.N, 0.0, 0.0).cpu().numpy()
        with np.errstate(divide="ignore"):
            t = x / (1.0 - x)
        y = [mpmath.log(mp(v)) if v > 0.0 else mp("-inf") for v in t]
        lo, hi = bracket(y, lambda L: par[0] + par[1] * L)
    elif kind == 18:                                        # scale * pow(e, 1 / shape)
        e = cb.rng_draws(seed, 1, rc.N, 1.0, 0.0).cpu().numpy()
        r = 1.0 / par[0]
        y = [mp_pow(float(v), r) for v in e]
        lo, hi = bracket(y, lambda P: par[1] * P)
    elif kind == 19:                                        # mode / pow(u, 1 / shape)
        u = cb.rng_draws(seed, 3, rc.N, 0.0, 0.0).cpu().numpy()
        r = 1.0 / par[0]
        y = [mp_pow(float(v), r) for v in u]
        lo, hi = bracket(y, lambda P: par[1] / P)
    else:                                                   # gamma(shape < 1): scale * (std_gamma(shape + 1) * pow(u, 1 / shape))
        shape, scale = (par[0], par[1]) if kind == 15 else (par[0] / 2.0, 2.0)
        g, u = rc.gamma_parts(host, seed, shape)
        r = 1.0 / shape
        y = [mp_pow(float(v), r) for v in u]
        lo, hi = bracket(y, lambda P: scale * (g * P))
    assert_inside(dev, lo, hi, rc.IDS[i])


@pytest.mark.parametrize("i", LIBM_COMPOSITE, ids=[rc.IDS[i] for i in LIBM_COMPOSITE])
def test_F_and_t_with_pow_inside_stay_close_to_the_host_build(cb, host, i):
    if not exact_ok(i):
        pytest.skip(f"a log comparison within {MARGIN_ULP} ulp of a tie on the host build")
    dev = device(cb, i)
    want = rc.host_sweep(host, i)["general"]
    with np.errstate(invalid="ignore"):
        rel = np.abs(dev - want) <= 16 * np.finfo(np.float64).eps * np.abs(want)
    same = rel | (dev == want) | (np.isnan(dev) & np.isnan(want))
    bad = np.flatnonzero(~same)
    assert bad.size == 0, (bad[:5], dev[bad[:3]], want[bad[:3]])


def x86_unsigned(q):
    """gcc's (unsigned)q on x86-64: the 64-bit truncation's low word, 0 from 2^63 on."""
    return int(q) & 0xFFFFFFFF if abs(q) < 2.0**63 else 0


@pytest.mark.parametrize("i", GEOMETRIC, ids=[rc.IDS[i] for i in GEOMETRIC])
def test_geometric_counts_are_the_reference_counts(cb, ref, i):
    kind, par = rc.CASES[i]
    m, p = (1, par[0]) if kind == 25 else (int(par[0]), par[1])
    dev = device(cb, i)
    e = cb.rng_draws(rc.case_seed(i), 1, rc.N * m, 1.0, 0.0).cpu().numpy().reshape(rc.N, m)
    denom = -math.log(1.0 - p) if p < 1.0 else math.inf      # glibc's log, as the reference has it (log(0) = -inf)
    denom_mp = -mpmath.log(1 - mpmath.mpf(p))
    want, loose = [], []
    for row in e:
        f, near = 0, False
        for x in row:
            q = float(x) / denom
            c = x86_unsigned(math.ceil(q))
            f = (f + c - 1) & 0xFFFFFFFF if kind != 25 else c
            exact = mpmath.mpf(float(x)) / denom_mp
            near |= abs(exact - mpmath.nint(exact)) <= 4 * math.ulp(q) and q != 0.0
        want.append(float(f))
        loose.append(near)
    want, loose = np.array(want), np.array(loose)
    bad = np.flatnonzero((dev != want) & ~loose)
    assert bad.size == 0, (bad[:5], dev[bad[:3]], want[bad[:3]])
    if not loose.any():
        assert rc.stream_sha256(want) == GOLD[rc.IDS[i]]["sha256"]
    if p <= 1e-9:
        assert (want >= 2.0**31).any()                      # past 2^31 - and with p = 1e-12 wrapped past 2^32
    if ref is not None:
        live = np.array(rng_draws_ex(ref, "ref", rc.case_seed(i), kind, par, rc.N))
        assert np.flatnonzero((dev != live) & ~loose).size == 0


# ---- paths 2 and 3: the sweep as model code on the general engine and the static tier
@pytest.fixture(scope="module")
def sweep_models(cb, tmp_path_factory):
    d = tmp_path_factory.mktemp("random_sweep_model")
    rc.write_model_table(d)
    sys.path.insert(0, str(rc.ROOT / "scripts"))
    import build_model
    ids = {}
    for engine, src in zip(("general", "static"), rc.model_sources(d)):
        ids[engine] = cb.load_model(build_model.build(src, d / f"lib{src.stem}.so", ["-I", str(d)]))
    return ids


def run_model(cb, model_id):
    for i in range(len(rc.CASES)):
        proven(i)
    n = len(rc.MODEL_CASES)
    dev = torch.device("cuda", torch.cuda.current_device())
    ones = torch.ones(n, dtype=torch.float64, device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(ones, ones, num_objects=0, master_seed=rc.SEED, model=model_id, queue_spill_cap=4096, diag=diag)
    torch.cuda.synchronize()
    counters = res.counters.cpu().numpy().astype(np.uint64).tolist()
    rows = [(int(st), int(o), float(t), [int(c) for c in cs]) for st, o, t, cs in
            zip(res.status.cpu().tolist(), res.objects.cpu().tolist(), res.t_end.cpu().tolist(), counters)]
    return rows, int(diag[2].item())


def test_model_code_on_both_engines_draws_the_path_one_stream(cb, ref, host, sweep_models):
    got = {engine: run_model(cb, sweep_models[engine]) for engine in ("general", "static")}
    assert got["static"][1] == 0                                        # no trial handed to the general engine
    want = rc.expected_model_rows(lambda i, n: device(cb, i, n))
    for engine in ("general", "static"):
        rows = got[engine][0]
        for i, w in enumerate(want):
            status, objects, t_end, counters = rows[i]
            assert status == 0 and objects == w[1], (engine, rc.IDS[i], status)
            assert counters == w[0], (engine, rc.IDS[i])
            assert t_end == w[2], (engine, rc.IDS[i], t_end, w[2])       # the clock after the held durations is their sum
    flip = [r[:2] + (r[2], r[3]) for r in (got["general"][0][-1], got["static"][0][-1])]
    assert flip[0] == flip[1] and flip[1][0] == 0                       # a flip and an exponential in one sampler
    host_static = rc.host_model(host, 1)[-1]
    assert (host_static[3], host_static[4]) == (flip[1][2], flip[1][3])
    if ref is not None:                                                 # geometric past 2^32 on paths 2 and 3: the reference's
        for i, (kind, par) in enumerate(rc.CASES):
            if kind in rc.GEOMETRIC_KINDS and (par[0] if kind == 25 else par[1]) <= 1e-9:
                live = np.array(rng_draws_ex(ref, "ref", rc.case_seed(i), kind, par, rc.N))
                assert got["static"][0][i][3][0] == rc.model_counters(live)[0], rc.IDS[i]
