"""Golden vectors for examples/clinic_model.cuh (a walk-in clinic drawing every model-code cmb_random distribution, alias
triage, summaries), produced by the UNMODIFIED reference (oracle/_ref/libclinicdrv.so: the same clinic written against the
reference's API in oracle/ref_build/clinic_driver.c, built by oracle/clinic.mk).

    python tests/golden/make_clinic_golden.py      -> tests/golden/clinic_vectors.json

Per case num_objects (arrival groups), arr_mean, srv_mean; per trial (seed cmb_random_fmix64(MASTER, i)) events, objects,
t_end and sum_wait as hex floats, max_queue (patients sent home), the eight counters of each of the five summaries
(rows[report]) and the SHA-256 of the first `trace` pops (key, time) as tests/cmb_cases.py's trace_digest forms it.  Used by
tests/test_model_random.py (both engines' source text on the CPU) and tests/test_gpu_clinic.py (both user libraries)."""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "tests"))
from clinic_cases import REPORTS, load_clinic_ref, ref_run, ref_trace   # noqa: E402
from cmb_cases import TRACE, trace_digest                                # noqa: E402
from oracle_libs import load_ref                                         # noqa: E402

MASTER = 0x34F05C64D7AD598F
CASES = [
    # name, num_objects, arr_mean, srv_mean, trials
    ("light", 400, 3.0, 0.5, 6),
    ("busy", 600, 1.6, 0.6, 6),        # desk 0 near saturation: long queues
    ("slow_desks", 300, 2.0, 1.0, 5),
    ("short", 40, 2.0, 1.0, 5),
]


def main():
    lib = load_clinic_ref()
    assert lib is not None, "oracle/_ref/libclinicdrv.so is not built (make -C oracle all && make -C oracle -f clinic.mk)"
    fmix64 = load_ref().ref_fmix64
    out = {"master": MASTER, "trace": TRACE, "cases": []}
    for name, nobj, arr, srv, n in CASES:
        per_report = [ref_run(lib, MASTER, 0, n, nobj, arr, srv, rep) for rep in range(len(REPORTS))]
        trials = []
        for i, r in enumerate(per_report[0]):
            _, keys, times = ref_trace(lib, fmix64(MASTER, i), nobj, arr, srv, 0, TRACE)
            trials.append({"events": r.events, "objects": r.objects, "t_end": float(r.t_end).hex(),
                           "sum_wait": float(r.sum_wait).hex(), "max_queue": r.max_queue,
                           "rows": [list(per_report[rep][i].counter) for rep in range(len(REPORTS))],
                           "trace_sha256": trace_digest(keys, times, r.events)})
        out["cases"].append({"name": name, "num_objects": nobj, "arr_mean": float(arr).hex(), "srv_mean": float(srv).hex(),
                             "trials": trials})
        print(name, nobj, [t["events"] for t in trials], [t["objects"] for t in trials])
    (ROOT / "tests/golden/clinic_vectors.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
