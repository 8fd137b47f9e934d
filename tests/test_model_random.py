"""CPU tests of the cmb_random distributions, alias tables and summaries that model code calls (cimba_b200/csrc/distributions.cuh,
summary.cuh, the names in cmb_device.cuh), and of examples/clinic_model.cuh, which draws every one of them.

The source text is compiled for the host (tests/model_random_host.cpp):
  * each distribution drawn through the general path's formulation and through the static tier's, the latter as the dispatcher
    draws a sampler (rectangles only, and on giving up the generator rewound and the draw repeated): the same stream, bit for bit;
  * cmb_random_loaded_dice and cmb_random_hyperexponential never index past n - 1, even above probabilities that sum to 1 - 2^-40;
  * cmb_random_alias_create's tables equal the C ABI's cimba_b200_alias_create, and the summary calls its cimba_b200_*summary_*;
  * the clinic on the general engine and on the static tier against the vectors of the same clinic written against the
    unmodified reference (tests/golden/clinic_vectors.json, oracle/ref_build/clinic_driver.c): every trial the same in events,
    objects, clock, sums, patients sent home, all eight counters (each of its five summaries in turn) and the pop trace.
The static kernel of the clinic is compiled for sm_90a and its ptxas report read (no GPU needed)."""
import ctypes as C
import random
import re
import struct
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from clinic_cases import GOLD as CLINIC_GOLD, LOGPOW_REPORTS, REPORTS, load_clinic_ref, ref_run
from cmb_cases import TRACE, trace_digest

ROOT = Path(__file__).resolve().parents[1]
MASTER = 0x34F05C64D7AD598F
KINDS = ["std_exponential", "triangular", "lognormal", "logistic", "cauchy", "hypoexponential", "hyperexponential", "std_gamma",
         "gamma_shape_below_1", "gamma", "std_beta", "beta", "PERT_mod", "weibull", "pareto", "chisquared", "F_dist", "std_t_dist",
         "t_dist", "rayleigh", "geometric", "binomial", "negative_binomial", "poisson", "loaded_dice", "alias_sample",
         "chisquared_1"]
ZIGGURAT_KINDS = {0, 2, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 15, 16, 17, 18, 19, 20, 22, 23, 26}


class HostResult(C.Structure):
    _fields_ = [("events", C.c_uint64), ("objects", C.c_uint64), ("t_end", C.c_double), ("sum_wait", C.c_double),
                ("max_fel", C.c_uint64), ("max_queue", C.c_uint64), ("counter", C.c_uint64 * 8), ("status", C.c_uint32),
                ("pad", C.c_uint32)]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = tmp_path_factory.mktemp("model_random") / "libmodel_random_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                    "-shared", "-fPIC", str(ROOT / "tests/model_random_host.cpp"), "-o", str(so)], check=True, capture_output=True)
    lib = C.CDLL(str(so))
    lib.host_random_streams.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                        C.POINTER(C.c_uint64)]
    lib.host_dice_bound.argtypes = [C.c_uint, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_uint),
                                    C.POINTER(C.c_double)]
    lib.host_alias_create.argtypes = [C.c_uint, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    lib.host_summaries.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                   C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
    lib.host_clinic_run_trials.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.c_double,
                                           C.c_double, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double),
                                           C.POINTER(HostResult)]
    assert lib.host_random_kinds() == len(KINDS)
    return lib


def _ptr(a, t):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.mark.parametrize("kind", range(len(KINDS)), ids=KINDS)
def test_static_tier_draws_the_general_paths_stream(host, kind):
    """20 000 variates from one seed: the static tier's inline formulation, tried with the rectangles first as a sampler is,
    equals the general path's (the rnd_* functions cimba_b200_rng_draws_ex runs) bit for bit; the ziggurat kinds do give up on
    the rectangles now and then, and every such draw still ends."""
    n = 20_000
    gen, st = np.zeros(n), np.zeros(n)
    rewinds = C.c_uint64(0)
    assert host.host_random_streams(kind, 0x9E3779B97F4A7C15 + kind, n, _ptr(gen, C.c_double), _ptr(st, C.c_double),
                                    C.byref(rewinds)) == 0
    assert gen.view(np.uint64).tolist() == st.view(np.uint64).tolist()
    assert (rewinds.value > 0) == (kind in ZIGGURAT_KINDS), rewinds.value
    assert np.isfinite(gen).all()


def test_loaded_dice_and_hyperexponential_stay_inside_the_arrays(host):
    """Probabilities that sum to 1 - 2^-40 (the reference accepts them) and the largest uniform below 1, which lies above that
    sum: the face is the last one with a positive probability, and the hyperexponential reads its mean, never the sentinel."""
    for pa in ([0.5, 0.25, 0.25 - 2.0**-40], [0.5, 0.5 - 2.0**-40, 0.0], [1.0 - 2.0**-40]):
        n = len(pa)
        assert sum(pa) < 1.0 and abs(sum(pa) - 1.0) < 1e-3
        p = np.array(pa)
        ma = np.array([1.0 + i for i in range(n)] + [float("nan")])
        face, hyper = C.c_uint(0), C.c_double(0.0)
        host.host_dice_bound(n, _ptr(p, C.c_double), _ptr(ma, C.c_double), C.byref(face), C.byref(hyper))
        want = max(i for i in range(n) if pa[i] > 0.0)
        assert face.value == want, (pa, face.value)
        assert hyper.value == ma[want], (pa, hyper.value)
    ma = np.array([float("nan")])        # n = 0: face 0 and no mean read
    face, hyper = C.c_uint(7), C.c_double(1.0)
    host.host_dice_bound(0, _ptr(ma, C.c_double), _ptr(ma, C.c_double), C.byref(face), C.byref(hyper))
    assert face.value == 0 and hyper.value == 0.0


def test_alias_create_in_model_code_equals_the_c_abi(host, cb):
    """cmb_random_alias_create's tables equal cimba_b200_alias_create's for random probability vectors of 1..64 entries."""
    from cimba_b200 import _lib
    raw = C.CDLL(str(_lib.LIB_PATH))
    raw.cimba_b200_alias_create.argtypes = [C.c_uint32, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    rnd = np.random.default_rng(20261017)
    for trial in range(300):
        n = int(rnd.integers(1, 65))
        w = rnd.random(n) ** 3
        if trial % 7 == 0:
            w[rnd.integers(0, n)] = 0.0
        if w.sum() == 0.0:
            w[0] = 1.0
        p = w / w.sum()
        u1, a1 = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
        u2, a2 = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
        assert host.host_alias_create(n, _ptr(p, C.c_double), _ptr(u1, C.c_uint64), _ptr(a1, C.c_uint32)) == 0
        assert raw.cimba_b200_alias_create(n, _ptr(p, C.c_double), _ptr(u2, C.c_uint64), _ptr(a2, C.c_uint32)) == 0
        assert u1.tolist() == u2.tolist() and a1.tolist() == a2.tolist(), (trial, n)
    p = np.full(65, 1.0 / 65)
    u, al = np.zeros(65, np.uint64), np.zeros(65, np.uint32)
    for n in (0, 65):                   # no entries, or more than the table's capacity of 64: refused (model code flags the trial)
        assert host.host_alias_create(n, _ptr(p, C.c_double), _ptr(u, C.c_uint64), _ptr(al, C.c_uint32)) == -1, n


def _bits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def test_summary_calls_equal_the_c_abi(host, cb):
    """cmb_datasummary_* / cmb_wtdsummary_* in model code equal cimba_b200_datasummary_* / _wtdsummary_* on the host bit for
    bit (add, merge, count, min, max, mean, variance, stddev, skewness, kurtosis), and cmb_summary_to_counters writes the row."""
    from cimba_b200 import _lib
    raw = C.CDLL(str(_lib.LIB_PATH))
    DS, WS = _lib.DataSummaryStruct, _lib.WtdSummaryStruct
    for name in ("mean", "variance", "stddev", "skewness", "kurtosis"):
        getattr(raw, f"cimba_b200_datasummary_{name}").restype = C.c_double
        getattr(raw, f"cimba_b200_wtdsummary_{name}").restype = C.c_double
    raw.cimba_b200_datasummary_add.argtypes = [C.POINTER(DS), C.c_double]
    raw.cimba_b200_wtdsummary_add.argtypes = [C.POINTER(WS), C.c_double, C.c_double]
    rnd = np.random.default_rng(7)
    for weighted in (0, 1):
        for n in (1, 2, 3, 4, 17, 1000):
            x = rnd.standard_cauchy(n)
            w = rnd.random(n)
            if n > 3:
                w[3] = 0.0                      # a zero weight is skipped
            k = n // 3
            out, row = np.zeros(13), np.zeros(8, np.uint64)
            host.host_summaries(weighted, n, k, _ptr(x, C.c_double), _ptr(w, C.c_double), _ptr(out, C.c_double),
                                _ptr(row, C.c_uint64))
            if weighted:
                a, b, c = WS(), WS(), WS()
                for s in (a, b):
                    raw.cimba_b200_wtdsummary_initialize(C.byref(s))
                for i in range(n):
                    raw.cimba_b200_wtdsummary_add(C.byref(a if i < k else b), x[i], w[i])
                raw.cimba_b200_wtdsummary_merge(C.byref(c), C.byref(a), C.byref(b))
                base, wsum, pre = c.base, c.wsum, "cimba_b200_wtdsummary_"
            else:
                a, b, c = DS(), DS(), DS()
                for s in (a, b):
                    raw.cimba_b200_datasummary_initialize(C.byref(s))
                for i in range(n):
                    raw.cimba_b200_datasummary_add(C.byref(a if i < k else b), x[i])
                raw.cimba_b200_datasummary_merge(C.byref(c), C.byref(a), C.byref(b))
                base, wsum, pre = c, float(c.count), "cimba_b200_datasummary_"
            want = [float(base.count), base.min, base.max, base.m1, base.m2, base.m3, base.m4, wsum if weighted else 0.0]
            want += [getattr(raw, pre + s)(C.byref(c)) for s in ("mean", "variance", "stddev", "skewness", "kurtosis")]
            assert [_bits(v) for v in out] == [_bits(v) for v in want], (weighted, n)
            assert row.tolist() == [base.count] + [_bits(v) for v in (base.min, base.max, base.m1, base.m2, base.m3, base.m4, wsum)]


# ---- the clinic on both engines, against the reference's vectors
GENERAL, STATIC = 0, 1


def run_clinic(host, engine, nobj, arr, srv, report, first, n, trace=TRACE):
    out = (HostResult * n)()
    keys = (C.c_uint64 * max(1, n * trace))()
    times = (C.c_double * max(1, n * trace))()
    assert host.host_clinic_run_trials(engine, MASTER, first, n, nobj, arr, srv, float(report), 1 << 26, trace, keys, times,
                                       out) == 0
    rows = []
    for i in range(n):
        o = out[i]
        h = trace_digest(np.ctypeslib.as_array(keys)[i * trace:(i + 1) * trace],
                         np.ctypeslib.as_array(times)[i * trace:(i + 1) * trace], o.events) if trace else ""
        rows.append((o.status, o.events, o.objects, o.t_end.hex(), o.sum_wait.hex(), o.max_queue, list(o.counter), h))
    return rows


def check_logpow_row(got, want, what):
    """A summary of logistic / weibull / pareto / gamma-below-1 values: the count exactly, each of min, max and the moments
    within 4 eps of the largest magnitude among the pair (CUDA's log / pow against glibc's; on the CPU both are glibc's)."""
    assert got[0] == want[0], what
    for k in range(1, 8):
        g, w = _double(got[k]), _double(want[k])
        assert abs(g - w) <= 4 * np.finfo(float).eps * max(abs(g), abs(w)), (what, k, g, w)


def _double(u):
    return struct.unpack("<d", struct.pack("<Q", int(u)))[0]


@pytest.mark.parametrize("report", range(len(REPORTS)), ids=REPORTS)
@pytest.mark.parametrize("engine", [GENERAL, STATIC], ids=["general", "static"])
@pytest.mark.parametrize("case", CLINIC_GOLD["cases"], ids=[c["name"] for c in CLINIC_GOLD["cases"]])
def test_clinic_matches_the_reference_vectors(host, case, engine, report):
    """Every vector trial of tests/golden/clinic_vectors.json (the clinic written against the unmodified reference):
    events, patients served, clock, time in clinic, patients sent home, the pop trace, and all eight counters of the summary
    `report` - exactly; the log / pow summaries within 4 eps (they are exact here, both sides using glibc).  Status 0."""
    n = len(case["trials"])
    got = run_clinic(host, engine, case["num_objects"], float.fromhex(case["arr_mean"]), float.fromhex(case["srv_mean"]),
                     report, 0, n, CLINIC_GOLD["trace"])
    for i, (g, w) in enumerate(zip(got, case["trials"])):
        what = (case["name"], engine, report, i)
        assert g[0] == 0, what
        assert g[1:6] == (w["events"], w["objects"], w["t_end"], w["sum_wait"], w["max_queue"]), what
        assert g[7] == w["trace_sha256"], (what, "pop trace")
        if report in LOGPOW_REPORTS:
            check_logpow_row(g[6], w["rows"][report], what)
        else:
            assert g[6] == w["rows"][report], what


def test_the_clinic_vectors_exercise_what_they_claim():
    """Every trial sends patients home and serves some; groups of more than one patient and more than one visit code occur;
    the busy case queues at desk 0."""
    for case in CLINIC_GOLD["cases"]:
        for t in case["trials"]:
            assert t["max_queue"] > 0 and t["objects"] > 0
            assert _double(t["rows"][3][2]) > 1.0 and _double(t["rows"][4][2]) >= 2.0     # largest group, largest visit code
    busy = next(c for c in CLINIC_GOLD["cases"] if c["name"] == "busy")
    assert max(_double(t["rows"][0][2]) for t in busy["trials"]) >= 5.0                  # desk 0's longest queue


def test_clinic_on_drawn_parameters(host):
    """Drawn means, sizes and first trials: the static tier equals the general engine, and both equal the live reference
    build (oracle/_ref/libclinicdrv.so) where it was built."""
    ref = load_clinic_ref()
    rnd = random.Random(20261017)
    for _ in range(8):
        nobj, arr, srv = rnd.randint(5, 300), rnd.choice([1.2, 2.0, 3.5]), rnd.choice([0.3, 0.5, 0.9])
        report, first = rnd.randrange(5), rnd.randint(0, 10_000)
        static = run_clinic(host, STATIC, nobj, arr, srv, report, first, 5, 0)
        assert static == run_clinic(host, GENERAL, nobj, arr, srv, report, first, 5, 0)
        if ref is not None:
            want = ref_run(ref, MASTER, first, 5, nobj, arr, srv, report)
            for g, w in zip(static, want):
                assert g[:6] == (0, w.events, w.objects, w.t_end.hex(), w.sum_wait.hex(), w.max_queue), (nobj, arr, srv, first)
                if report in LOGPOW_REPORTS:
                    check_logpow_row(g[6], list(w.counter), (nobj, arr, srv, first))
                else:
                    assert g[6] == list(w.counter), (nobj, arr, srv, first)
    if ref is None:
        pytest.skip("oracle/_ref/libclinicdrv.so not built (needs the reference sources): static = general checked only")


# ---- the static kernel's build report (no GPU needed)
SRC = """#include "cmb_launch.cuh"
#include "../../examples/clinic_model.cuh"
namespace cimba_b200 { namespace cmb {
template __global__ void static_trial_kernel<clinic_example::ClinicT, 4, 2, 0, false>(const StaticArgs);
}}
"""


def test_clinic_static_kernel_build_report(tmp_path):
    """ptxas on sm_90a: the clinic's static kernel builds, with no more registers, stack frame and spills than CUDA 12.9 gives it
    today (168 registers, 968 bytes of stack frame, 716 / 316 bytes of spill stores / loads), so that a regression in the
    inlined distributions fails here.  They are not zero: every
    distribution inlines into the dispatcher, the sampler's three branches and the body's ten draws among them, under the
    tier's occupancy bound; and the Vose tables are built and read, and the model's arrays (hyperexponential means, dice
    probabilities) read, at run-time indices, so the model struct lives in local memory."""
    sys.path.insert(0, str(ROOT))
    import __graft_entry__ as g
    (tmp_path / "k.cu").write_text(SRC)
    flags = [f for f in g.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    cmd = [g._nvcc(), *flags, "-Xptxas", "-v", "-I", str(g.CSRC), "-I", str(ROOT / "include"), "-cubin", "-o",
           str(tmp_path / "k.cubin"), str(tmp_path / "k.cu")]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    m = re.search(r"Compiling entry function '\w*static_trial_kernel\w*' for 'sm_90a'\n(.*?)(?=ptxas info\s+: Compile time)",
                  p.stderr, re.S)
    assert m, p.stderr
    text = m.group(1)
    stack = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    regs = re.search(r"Used (\d+) registers", text)
    assert stack and regs, text
    print(f"ClinicT static kernel: {regs.group(1)} registers, {stack.group(1)} bytes stack frame, "
          f"{stack.group(2)} / {stack.group(3)} bytes spill stores / loads")
    assert int(regs.group(1)) <= 168 and int(stack.group(1)) <= 968, text
    assert int(stack.group(2)) <= 716 and int(stack.group(3)) <= 316, text
