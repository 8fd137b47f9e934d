"""Golden vectors for examples/repair_model.cuh (a machine shop: a repair crew pool, an inspection bench), produced by the
UNMODIFIED reference (oracle/_ref/librepairdrv.so: the same shop written against the reference's API in
oracle/ref_build/repair_driver.c, built by oracle/repair.mk).

    python tests/golden/make_repair_golden.py      -> tests/golden/repair_vectors.json

The format of make_cmb_golden.py: per case servers, num_objects, arr_mean, srv_mean, params (machines, exit while holding);
per trial (seed cmb_random_fmix64(MASTER, i)) events, objects, t_end and sum_wait as hex floats, all eight counters and the
SHA-256 of the first `trace` pops (key, time).  Used by tests/test_static_resources.py (the static tier's and the general
engine's source text run on the CPU) and tests/test_gpu_static_resources.py (both on the device).

Eight machines claim one or two units; with four or fewer crew, the claims can deadlock: four two-unit claimants each
keep the one unit they grabbed and wait for another that never comes.  The reference's trial then ends when its event
list runs dry, and so does the port's (case "deadlock").  The other cases have more crew than two-unit claimants."""
import hashlib
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "tests"))
from oracle_libs import load_ref                               # noqa: E402
from repair_cases import load_repair_ref, ref_run, ref_trace   # noqa: E402

MASTER = 0x34F05C64D7AD598F
TRACE = 2000
CASES = [
    # name, servers, num_objects, arr_mean, srv_mean, params, trials
    ("moderate", 5, 2000, 4.0, 1.0, [8, 0], 6),
    ("saturated", 5, 2000, 1.5, 1.0, [8, 0], 6),          # a busy crew: many partial grabs
    ("light", 6, 1500, 8.0, 1.0, [8, 0], 5),
    ("crew_of_one", 1, 2000, 5.0, 1.0, [8, 0], 5),
    ("five_machines", 3, 1000, 3.0, 1.0, [5, 0], 5),      # fewer machines than the static tier's eight slots
    ("twelve_machines", 7, 500, 4.0, 1.0, [12, 0], 4),    # more than it holds: the general engine's
    ("exit_holding", 5, 500, 4.0, 1.0, [8, 1], 4),        # the last cycle exits with the crew held: the general engine's
    ("deadlock", 2, 2000, 1.5, 1.0, [8, 0], 4),           # two-unit claims each holding one unit wait for ever
]


def main():
    lib = load_repair_ref()
    assert lib is not None, "oracle/_ref/librepairdrv.so is not built (make -C oracle all && make -C oracle -f repair.mk)"
    fmix64 = load_ref().ref_fmix64
    out = {"master": MASTER, "trace": TRACE, "cases": []}
    for name, servers, nobj, arr, srv, params, n in CASES:
        res = ref_run(lib, servers, MASTER, 0, n, nobj, arr, srv, params)
        trials = []
        for i, r in enumerate(res):
            _, keys, times = ref_trace(lib, servers, fmix64(MASTER, i), nobj, arr, srv, params, TRACE)
            h = hashlib.sha256(np.array(keys, dtype=np.uint64).tobytes() + np.array(times, dtype=np.float64).tobytes())
            trials.append({"events": r.events, "objects": r.objects, "t_end": float(r.t_end).hex(),
                           "sum_wait": float(r.sum_wait).hex(), "counters8": list(r.counter), "pops": len(keys),
                           "trace_sha256": h.hexdigest()})
        out["cases"].append({"name": name, "servers": servers, "num_objects": nobj, "arr_mean": float(arr).hex(),
                             "srv_mean": float(srv).hex(), "params": params, "trials": trials})
        print(name, servers, nobj, [t["events"] for t in trials], [t["counters8"][:2] for t in trials])
    (ROOT / "tests/golden/repair_vectors.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
