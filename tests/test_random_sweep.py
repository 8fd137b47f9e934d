"""CPU side of the cmb_random parameter sweep (tests/random_sweep_cases.py): every case through the host build of the
formulation the device runs (tests/random_sweep_host.cpp compiles cimba_b200/csrc/distributions.cuh for the CPU).

  * every case sits inside the reference's domain, and inside its work bound: the host build's generator calls stay under
    N * calls_bound, and N * calls_bound under one launch's budget - proven here before any GPU test draws the case;
  * the general path's stream equals the plain-C port's (oracle/port) and the unmodified reference build's where it was built,
    bit for bit (a NaN as a NaN: the payloads of x86 and CUDA differ);
  * the sweep as model code (tests/random_sweep_model.cuh) on the general engine and on the static tier's dispatcher (sampled
    holds rectangles first, on giving up the generator and the flip cache rewound and the sampler repeated) gives the
    counters of the general path's stream, and the static tier's clock is the sum of the held durations;
  * the Marsaglia-Tsang log comparisons of at least 90 % of the gamma-family cases stay more than MARGIN_ULP from a tie, so that
    the GPU tests demand bit-exactness of most of them;
  * tests/golden/random_sweep_vectors.json is fresh: its cases, hashes, call counts and margins are what the table and the
    host build give today."""
import json
import math

import numpy as np
import pytest

import random_sweep_cases as rc
from oracle_libs import load_port, load_ref, rng_draws_ex

GOLD_PATH = rc.ROOT / "tests/golden/random_sweep_vectors.json"
MARGIN_ULP = 16.0


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return rc.build_host(tmp_path_factory.mktemp("random_sweep"))


@pytest.fixture(scope="module")
def swept(host):
    return [rc.host_sweep(host, i) for i in range(len(rc.CASES))]


@pytest.fixture(scope="module")
def gold():
    return json.loads(GOLD_PATH.read_text())


def same_bits(a, b):
    return np.array_equal(rc.canonical(a).view(np.uint64), rc.canonical(b).view(np.uint64))


def test_every_case_is_inside_the_reference_domain_and_the_launch_budget():
    assert len(set(rc.IDS)) == len(rc.CASES)
    assert {k for k, _ in rc.CASES} == set(range(9, 34))
    total = 0
    for (kind, par), cid in zip(rc.CASES, rc.IDS):
        assert rc.in_domain(kind, par), cid
        assert rc.N * rc.calls_bound(kind, par) <= rc.LAUNCH_CALLS, cid
        total += rc.N * rc.calls_bound(kind, par)
    assert total <= rc.LAUNCH_CALLS, total           # all cases in one launch fit too
    model = sum(rc.N * rc.calls_bound(k, p) * (2 if rc.held_ok(k, p) else 1) for k, p in rc.CASES)
    assert model <= rc.LAUNCH_CALLS, model           # the sweep model's launch: every case, held cases twice


def test_the_grid_crosses_the_branch_edges():
    shapes = {p[0] for k, p in rc.CASES if k == 31}
    assert {1e-300, 0.3, 1.0 / 3.0, 0.34, 1.0, 1e6} <= shapes
    assert {p[0] for k, p in rc.CASES if k == 25} >= {1e-12, 1e-9, 1.0}
    assert min(p[0] for k, p in rc.CASES if k == 20) < 2.0 and min(p[2] for k, p in rc.CASES if k == 22) < 1.0
    assert {p[3] for k, p in rc.CASES if k == 32} >= {1e-6, 1e3}
    assert any(k == 29 and math.fsum(p[1:]) == 1.0 - 2.0**-40 for k, p in rc.CASES)


@pytest.mark.parametrize("i", range(len(rc.CASES)), ids=rc.IDS)
def test_host_build_finishes_each_case_within_its_work_bound(swept, i):
    kind, par = rc.CASES[i]
    assert swept[i]["calls"] <= rc.N * rc.calls_bound(kind, par), swept[i]["calls"] / rc.N


@pytest.mark.parametrize("i", range(len(rc.CASES)), ids=rc.IDS)
def test_general_path_equals_port_and_reference(swept, ref, i):
    kind, par = rc.CASES[i]
    gen = swept[i]["general"]
    port = np.array(rng_draws_ex(load_port(), "port", rc.case_seed(i), kind, par, rc.N))
    assert same_bits(gen, port), np.flatnonzero(rc.canonical(gen).view(np.uint64) != rc.canonical(port).view(np.uint64))[:5]
    if ref is not None:
        assert same_bits(gen, np.array(rng_draws_ex(ref, "ref", rc.case_seed(i), kind, par, rc.N)))


@pytest.fixture(scope="module")
def model_rows(host):
    return {"general": rc.host_model(host, 0), "static": rc.host_model(host, 1)}


def test_held_cases_are_finite_nonnegative_durations(host):
    """Every case the sweep model also draws as sampled holds gives 2N finite variates >= 0 whose running sum stays finite,
    proven here before a GPU test runs the model."""
    for i, (kind, par) in enumerate(rc.CASES):
        if rc.held_ok(kind, par):
            v = rc.host_sweep(host, i, 2 * rc.N)["general"]
            assert np.isfinite(v).all() and (v >= 0.0).all() and np.isfinite(np.cumsum(v[rc.N:])).all(), rc.IDS[i]
    assert sum(rc.held_ok(k, p) for k, p in rc.CASES) >= 0.6 * len(rc.CASES)


@pytest.fixture(scope="module")
def model_want(host):
    return rc.expected_model_rows(lambda i, n: rc.host_sweep(host, i, n)["general"])


@pytest.mark.parametrize("i", range(len(rc.CASES)), ids=rc.IDS)
def test_static_tier_give_up_and_rewind_equals_general_path(model_rows, model_want, i):
    """Case i of the sweep model (tests/random_sweep_model.cuh) on the general engine and on the static tier - the tier's own
    dispatcher, sampled holds tried with the rectangles only and repeated after a rewind - gives the counters of the general
    path's stream, status 0, and a clock equal to the sum of the held durations."""
    w = model_want[i]
    for engine in ("general", "static"):
        status, events, objects, t_end, counters = model_rows[engine][i]
        assert status == 0 and objects == w[1], engine
        assert counters == w[0], engine
        assert t_end == w[2], (engine, t_end, w[2])


def test_sweep_model_flip_sampler_rewinds_the_flip_cache(model_rows):
    """Kind 100: a sampler that calls cmb_random_flip() and then draws an exponential.  When the exponential gives up on the
    rectangles, the static tier puts back the flip cache with the generator, so its stream is the general engine's."""
    g, s = model_rows["general"][-1], model_rows["static"][-1]
    assert rc.MODEL_CASES[-1][0] == 100 and s[0] == 0
    assert s == g


def test_gamma_family_margins_leave_most_cases_bit_exact(swept):
    fam = [i for i, (k, _) in enumerate(rc.CASES) if k in rc.GAMMA_FAMILY]
    assert all(swept[i]["compares"] > 0 for i in fam)              # every one of them reaches the log comparison
    ok = [i for i in fam if swept[i]["margin"] > MARGIN_ULP]
    assert len(ok) >= 0.9 * len(fam), [rc.IDS[i] for i in fam if i not in ok]


def test_golden_file_is_fresh(swept, gold):
    """The committed vectors belong to this table and this formulation (regenerate with
    tests/golden/make_random_sweep_golden.py after changing either)."""
    assert gold["seed"] == rc.SEED and gold["n"] == rc.N
    assert [c["id"] for c in gold["cases"]] == rc.IDS
    for i, c in enumerate(gold["cases"]):
        kind, par = rc.CASES[i]
        assert (c["kind"], c["params"], c["seed"]) == (kind, [float(v).hex() for v in par], rc.case_seed(i)), c["id"]
        s = swept[i]
        assert c["sha256"] == rc.stream_sha256(rc.canonical(s["general"])), c["id"]
        assert (c["calls"], c["compares"]) == (s["calls"], s["compares"]), c["id"]
        assert c["margin"] == (float(s["margin"]) if np.isfinite(s["margin"]) else None), c["id"]
        if rc.libm_value(kind, par):
            assert c["first"] == [float(v).hex() for v in s["general"][:len(c["first"])]], c["id"]


def test_geometric_wraps_past_two_to_the_32(swept):
    """At p = 1e-12 nearly every quotient passes 2^32: the reference's build keeps it modulo 2^32 (gcc's 64-bit conversion),
    so the stream holds no saturated 4294967295 and its values are spread over the whole unsigned range."""
    for i, (kind, par) in enumerate(rc.CASES):
        if kind == 25 and par[0] == 1e-12:
            v = swept[i]["general"]
            assert not (v == 4294967295.0).any() and v.max() > 2.0**31 and v.min() < 2.0**30
