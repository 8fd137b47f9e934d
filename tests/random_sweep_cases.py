"""The parameter sweep of every cmb_random distribution kind 9..33 (numbering of cimba_b200_rng_draws_ex / ref_rng_draws_ex),
shared by tests/test_random_sweep.py (CPU), tests/test_gpu_random_sweep.py (GPU) and tests/golden/make_random_sweep_golden.py.

Every case lies inside the domain the reference's release asserts describe (in_domain below), at the branch edges where a
kernel goes wrong: gamma's shape at 1 and 1/3, chisquared below 2, F / t below 1, geometric p down to 1e-12 (quotients past
2^32), PERT's lambda, probabilities that sum to 1 - 2^-40.  Each case carries a bound on the expected generator calls per
variate (calls_bound); a CPU test proves, on the host build of the same source text, that each case stays inside
N * calls_bound before any GPU test draws it, and that N * calls_bound stays under LAUNCH_CALLS for one launch."""
from __future__ import annotations

import ctypes as C
import hashlib
import itertools
import math
import subprocess
from pathlib import Path

import numpy as np

SEED = 0x5EED0F5EEDC0FFEE
N = 4096                        # variates per case (a multiple of 64: the reference's flip cache is empty between calls)
LAUNCH_CALLS = 1 << 24          # generator calls one launch may make, all cases of it together

GAMMA_SHAPES = [1e-300, 0.01, 0.3, 1.0 / 3.0, 0.34, 1.0 - 1e-6, 1.0, 1.0 + 1e-7, 2.5, 50.0, 1e6]
BETA_SHAPES = [0.05, 0.34, 1.0, 7.0]
P_GRID = [1e-12, 1e-9, 1e-6, 0.3, 0.5, 0.999, 1.0 - 2.0**-53, 1.0]
TINY = 5e-324                   # the smallest positive double: "zero" where the reference asserts > 0


def _cases():
    c = []
    for a in GAMMA_SHAPES:
        c.append((31, [a]))
        c.append((15, [a, 1.5]))
        c.append((20, [2.0 * a]))
    for a, b in itertools.product(BETA_SHAPES, BETA_SHAPES):
        c.append((16, [a, b, 0.0, 1.0]))
        c.append((21, [a, b]))
    for v in [0.05, 0.5, 1.0, 2.0, 30.0, 1e6]:
        c.append((22, [0.0, 1.0, v]))
    for p in P_GRID:
        c.append((25, [p]))
        c.append((27, [3, p]))
        c.append((33, [2, p]))
        c.append((26, [7, p]))
    for r in [1e-9, 0.01, 1.0, 20.0, 64.0]:
        c.append((28, [r]))
    for m, sd in [(0.0, TINY), (0.0, 1e-3), (700.0, 1.0), (-700.0, 1.0), (0.0, 30.0)]:
        c.append((10, [m, sd]))
    for mn, md, mx in [(0.0, 0.0, 1.0), (0.0, 1.0, 1.0), (0.0, TINY, 1.0), (0.0, 1.0 - 2.0**-53, 1.0), (1.0, 1.0, 1.0),
                       (-1e9, 0.0, 1e-9)]:
        c.append((9, [mn, md, mx]))
    for mn, md, mx, lam in [(0.0, 1e-9, 1.0, 4.0), (0.0, 1.0 - 1e-9, 1.0, 4.0), (0.0, TINY, 1.0, 4.0), (0.0, 0.5, 1.0, 1e-6),
                            (0.0, 0.25, 1.0, 1e-6), (0.0, 0.5, 1.0, 1e3), (0.0, 0.25, 1.0, 1e3)]:
        c.append((32, [mn, md, mx, lam]))
    c.append((17, [0.0, 1e-9, 1.0]))
    c.append((17, [-3.0, 2.0, 2.0 + 2.0**-51]))
    for m, s in [(0.0, 1.0), (1e3, 1e-3), (-5.0, 30.0)]:
        c.append((11, [m, s]))
    for sh in [0.01, 0.5, 1.0, 8.0, 1e3]:
        c.append((18, [sh, 2.0]))
        c.append((19, [sh, 1.0]))
    c += [(12, [0.0, 1.0]), (12, [0.0, 1e-300]), (23, [1.3]), (23, [1e-300]), (13, [1, 1e-300]), (13, [3, 0.5, 1.0, 2.0]),
          (24, [])]
    c += [(29, [3, 0.5, 0.25, 0.25 - 2.0**-40]), (29, [3, 0.0, 0.0, 1.0]), (29, [4, 0.0, 1.0 - 2.0**-40, 0.0, 0.0]),
          (29, [2, 0.5, 0.5])]
    c += [(14, [2, 1.0, 2.0, 0.5, 0.5 - 2.0**-40]), (14, [3, 1.0, 2.0, 3.0, 0.0, 1.0, 0.0]),
          (14, [3, 0.5, 1.0, 4.0, 0.0, 0.6, 0.4 - 2.0**-40])]
    c += [(30, [3, 0.0, 0.0, 1.0]), (30, [4, 0.25, 0.25, 0.25, 0.25]), (30, [3, 0.5, 0.25, 0.25 - 2.0**-40]),
          (30, [5, 0.0, 0.5, 0.0, 0.5, 0.0])]
    return c


NAMES = {9: "triangular", 10: "lognormal", 11: "logistic", 12: "cauchy", 13: "hypoexponential", 14: "hyperexponential",
         15: "gamma", 16: "beta", 17: "PERT", 18: "weibull", 19: "pareto", 20: "chisquared", 21: "F_dist", 22: "t_dist",
         23: "rayleigh", 24: "flip", 25: "geometric", 26: "binomial", 27: "negative_binomial", 28: "poisson", 29: "loaded_dice",
         30: "alias_sample", 31: "std_gamma", 32: "PERT_mod", 33: "pascal"}

CASES = _cases()
IDS = [f"{k:02d}-{NAMES[k]}({','.join(repr(float(v)) for v in p)})" for k, p in CASES]

# kinds whose draws run the Marsaglia-Tsang accept/reject loop, and so compare a log() with another expression
GAMMA_FAMILY = {15, 16, 17, 20, 21, 22, 31, 32}
# kinds whose values are unsigned counts (geometric quotients converted to unsigned)
GEOMETRIC_KINDS = {25, 27, 33}


def gamma_shapes(kind, p):
    """The shapes the case's draws pass to std_gamma's loop-free pow branch (shape < 1: std_gamma(shape + 1) * u^(1 / shape))."""
    if kind == 15:
        return [p[0]]
    if kind == 20:
        return [p[0] / 2.0]
    if kind == 21:
        return [p[0] / 2.0, p[1] / 2.0]
    if kind == 22:
        return [p[2] / 2.0]
    return []


def libm_value(kind, p):
    """True where the variate itself carries a log / pow result of the platform's libm (CUDA's on the device, glibc's in the
    reference): logistic, weibull, pareto, and every gamma draw whose shape is below 1 (gamma, chisquared, F, t)."""
    return kind in (11, 18, 19) or any(a < 1.0 for a in gamma_shapes(kind, p))


def held_ok(kind, p):
    """Cases whose every variate is a finite number >= 0, so that tests/random_sweep_model.cuh also draws them as the durations
    of sampled holds (tests/test_random_sweep.py proves it on the host build before a GPU test relies on it).  Out: kinds with
    negative values, and the cases that give NaN (std_gamma / beta below shape 1/3) or overflow (lognormal at mean 700,
    weibull and pareto at shape 0.01)."""
    if kind in (11, 12, 22):
        return False
    if kind == 9 and p[0] < 0.0 or kind == 16 and p[2] < 0.0 or kind in (17, 32) and p[0] < 0.0:
        return False
    if kind in (31, 16) and min(p[:1] if kind == 31 else p[:2]) <= 1.0 / 3.0:
        return False
    if kind == 10 and p[0] > 0.0 or kind in (18, 19) and p[0] < 0.1:
        return False
    return True


def _sums_to_one(pa):
    return abs(math.fsum(pa) - 1.0) <= 1e-3


def in_domain(kind, p):
    """The reference's release asserts (include/cmb_random.h, src/cmb_random.c), and the debug assert 0 < p <= 1 of geometric."""
    if kind == 9:
        return p[0] <= p[1] <= p[2]
    if kind in (10, 11):
        return p[1] > 0.0
    if kind in (12, 23):
        return p[-1] > 0.0
    if kind == 13:
        n = int(p[0])
        return n > 0 and len(p) == 1 + n and all(m > 0.0 for m in p[1:])
    if kind == 14:
        n = int(p[0])
        return n > 0 and len(p) == 1 + 2 * n and all(m > 0.0 for m in p[1:1 + n]) and _sums_to_one(p[1 + n:])
    if kind in (15, 18, 19):
        return p[0] > 0.0 and p[1] > 0.0
    if kind == 16:
        return p[0] > 0.0 and p[1] > 0.0 and p[2] < p[3]
    if kind == 17:
        return p[0] < p[1] < p[2]
    if kind == 20:
        return p[0] > 0.0
    if kind == 21:
        return p[0] > 0.0 and p[1] > 0.0
    if kind == 22:
        return p[1] > 0.0 and p[2] > 0.0
    if kind == 24:
        return True
    if kind == 25:
        return 0.0 < p[0] <= 1.0
    if kind in (26, 27, 33):
        return int(p[0]) > 0 and 0.0 < p[1] <= 1.0
    if kind == 28:
        return p[0] > 0.0
    if kind in (29, 30):
        n = int(p[0])
        return n > 0 and len(p) == 1 + n and all(v >= 0.0 for v in p[1:]) and _sums_to_one(p[1:])
    if kind == 31:
        return p[0] > 0.0
    if kind == 32:
        return p[0] < p[1] < p[2] and p[3] > 0.0
    return False


# expected generator calls per variate: a uniform is one call, a ziggurat exponential or normal at most 2 (1.02 on average),
# one Marsaglia-Tsang draw at most GAMMA_CALLS (normal + uniform per round, at least a third of the rounds accept)
EXP_CALLS = 2
GAMMA_CALLS = 12


def calls_bound(kind, p):
    if kind in (9, 11, 19, 24, 29):
        return 1
    if kind == 30:
        return 2
    if kind in (10, 18, 25):
        return EXP_CALLS
    if kind in (12, 23):
        return 2 * EXP_CALLS
    if kind == 13:
        return EXP_CALLS * int(p[0])
    if kind == 14:
        return 1 + EXP_CALLS
    if kind in (15, 20, 31):
        return GAMMA_CALLS + 1
    if kind in (16, 17, 21, 32):
        return 2 * (GAMMA_CALLS + 1)
    if kind == 22:
        return EXP_CALLS + GAMMA_CALLS + 1
    if kind == 26:
        return int(p[0])
    if kind in (27, 33):
        return EXP_CALLS * int(p[0])
    if kind == 28:
        return EXP_CALLS * (int(math.ceil(p[0])) + 2)
    raise ValueError(kind)


def case_seed(i):
    """The generator seed of case i: cmb_random_fmix64(SEED, i), the seed trial i of an experiment with master seed SEED gets."""
    m = (1 << 64) - 1
    h = (SEED + i) & m
    h ^= h >> 33
    h = (h * 0xFF51AFD7ED558CCD) & m
    h ^= h >> 33
    h = (h * 0xC4CEB9FE1A85EC53) & m
    return h ^ (h >> 33)


CANONICAL_NAN = np.array([0x7FF8000000000000], dtype="<u8").view(np.float64)[0]


def canonical(values):
    """The variates with every NaN replaced by one NaN: the reference's x86 NaNs and CUDA's carry different bits."""
    v = np.array(values, dtype=np.float64)
    v[np.isnan(v)] = CANONICAL_NAN
    return v


def stream_sha256(values):
    """SHA-256 of the variates' bit patterns, little-endian uint64 each."""
    return hashlib.sha256(np.ascontiguousarray(values, dtype=np.float64).view("<u8").tobytes()).hexdigest()


# ---- the sweep as model code (tests/random_sweep_model.cuh): every case, then kind 100 (a flip and an exponential in one sampler)
MODEL_CASES = CASES + [(100, [])]
MAXP = 8


def write_model_table(directory):
    """random_sweep_table.h for tests/random_sweep_model.cuh: the case table, parameters as exact hex literals."""
    rows = []
    for kind, par in MODEL_CASES:
        vals = [float(v) for v in par] + [0.0] * (MAXP - len(par))
        held = 1 if kind == 100 or held_ok(kind, par) else 0
        rows.append(f"    {{{kind}u, {len(par)}u, {held}u, {{{', '.join(v.hex() for v in vals)}}}}},")
    text = ("// generated by tests/random_sweep_cases.py (write_model_table): the cmb_random sweep's cases\n#pragma once\n"
            "#include <cstdint>\nnamespace random_sweep {\n"
            f"constexpr uint32_t NCASES = {len(MODEL_CASES)}u;\nconstexpr uint64_t NDRAW = {N}u;\nconstexpr uint32_t MAXP = {MAXP}u;\n"
            "struct Case { uint32_t kind, np, held; double p[MAXP]; };\n"
            "__device__ const Case CASES[NCASES] = {\n" + "\n".join(rows) + "\n};\n}  // namespace random_sweep\n")
    (Path(directory) / "random_sweep_table.h").write_text(text)
    return Path(directory)


FOLD_START = 0xCBF29CE484222325


def model_counters(body, held=None):
    """The eight counters tests/random_sweep_model.cuh writes for the body's variates and the held durations."""
    m = (1 << 64) - 1
    bits = np.ascontiguousarray(body, dtype=np.float64).view("<u8").tolist()

    def fold(bs):
        h = FOLD_START
        for b in bs:
            h = (((h ^ b) * 0x100000001B3) + 1) & m
        return h

    finite = np.asarray(body)[~np.isnan(body)]
    lo = float(finite.min()) if finite.size else math.inf
    hi = float(finite.max()) if finite.size else -math.inf
    as_bits = lambda x: int(np.array([x], dtype=np.float64).view("<u8")[0])
    held_bits = [] if held is None else np.ascontiguousarray(held, dtype=np.float64).view("<u8").tolist()
    return [fold(bits), bits[0], bits[-1], as_bits(lo), as_bits(hi), len(bits), int(np.isnan(body).sum()), fold(held_bits)]


def model_sources(directory):
    """The sweep model exported for the general engine and for the static tier (one process, no queue, and the one event slot the
    tier's form with the flip cache asks for), as .cu files."""
    d = Path(directory)
    head = (f'#include "{ROOT}/cimba_b200/csrc/cmb_launch.cuh"\n#include "{ROOT}/tests/random_sweep_model.cuh"\n')
    general, static = d / "random_sweep_general.cu", d / "random_sweep_static.cu"
    general.write_text(head + 'CMB_EXPORT_MODEL(random_sweep::SweepT<cimba_b200::cmb::Sim>, "cmb_random sweep, general engine")\n')
    static.write_text(head + 'CMB_EXPORT_STATIC_MODEL_EVENTS(random_sweep::SweepT, 1, 0, 1, "cmb_random sweep")\n')
    return general, static


# ---- the host build of the formulation (tests/random_sweep_host.cpp)
ROOT = Path(__file__).resolve().parents[1]
_D = C.POINTER(C.c_double)
_U = C.POINTER(C.c_uint64)


class HostResult(C.Structure):
    _fields_ = [("events", C.c_uint64), ("objects", C.c_uint64), ("t_end", C.c_double), ("sum_wait", C.c_double),
                ("counter", C.c_uint64 * 8), ("status", C.c_uint32), ("pad", C.c_uint32)]


def build_host(directory):
    so = Path(directory) / "librandom_sweep_host.so"
    write_model_table(directory)
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                    "-shared", "-fPIC", "-I", str(directory), str(ROOT / "tests/random_sweep_host.cpp"), "-o", str(so)],
                   check=True, capture_output=True)
    lib = C.CDLL(str(so))
    lib.sweep_draws.argtypes = [C.c_uint64, C.c_int, _D, C.c_uint32, C.c_uint64, _D, _U, _D, _U]
    lib.gamma_parts.argtypes = [C.c_uint64, C.c_double, C.c_uint64, _D, _D]
    lib.sweep_model_run.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.POINTER(HostResult)]
    return lib


def host_sweep(lib, i, n=N):
    """Case i on the host build of the general path's formulation: the stream, calls, margin and compares."""
    kind, par = CASES[i]
    gen = np.zeros(n)
    calls, margin, compares = C.c_uint64(), C.c_double(), C.c_uint64()
    p = (C.c_double * max(1, len(par)))(*[float(v) for v in par])
    rc = lib.sweep_draws(case_seed(i), kind, p, len(par), n, gen.ctypes.data_as(_D), C.byref(calls), C.byref(margin),
                         C.byref(compares))
    assert rc == 0, (i, kind, par)
    return {"general": gen, "calls": calls.value, "margin": margin.value, "compares": compares.value}


def host_model(lib, engine):
    """Every trial of the sweep model on the host build: engine 0 = the general engine, 1 = the static tier's dispatcher.
    Rows (status, events, objects, t_end bits, counters)."""
    out = (HostResult * len(MODEL_CASES))()
    assert lib.sweep_model_run(engine, SEED, len(MODEL_CASES), out) == 0
    return [(o.status, o.events, o.objects, o.t_end, list(o.counter)) for o in out]


def expected_model_rows(values_of):
    """What each trial of the sweep model must report, from a function that gives case i's first n variates of the general
    path's stream (path 1): counters, objects and the clock after the held durations (their sum, added in order)."""
    rows = []
    for i, (kind, par) in enumerate(CASES):
        held = held_ok(kind, par)
        v = values_of(i, 2 * N if held else N)
        t = 0.0
        if held:
            for x in v[N:]:
                t = t + float(x)
        rows.append((model_counters(v[:N], v[N:] if held else None), N, t))
    return rows


def gamma_parts(lib, seed, shape, n=N):
    """gamma's shape < 1 branch factor by factor: std_gamma(shape + 1) and the uniform after it, per variate."""
    g, u = np.zeros(n), np.zeros(n)
    lib.gamma_parts(seed, shape, n, g.ctypes.data_as(_D), u.ctypes.data_as(_D))
    return g, u

