"""Golden vectors for examples/event_model.cuh's EventTestT (the reference's own event-queue test, test/test_event.c), produced
by the UNMODIFIED reference (oracle/_ref/libeventdrv.so: test_events()'s sequence written against the reference's API in
oracle/ref_build/event_driver.c, built by oracle/event.mk).

    python tests/golden/make_event_golden.py      -> tests/golden/event_vectors.json

64 trials, trial i seeded fmix64(MASTER, i); trial 0's seed is the golden file's, 0x34f05c64d7ad598f (tests/event_cases.py).
Per trial: the seed, events executed, the final clock as a hex float, the eight counters and the whole pop trace (handle, time
as a hex float).  Used by tests/test_event_queue.py (both engines' source text on the CPU) and tests/test_gpu_event_queue.py."""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "tests"))
from event_cases import MASTER, TRACE_CAP, VECTORS, fmix64, load_event_ref, ref_run   # noqa: E402

TRIALS = 64


def main():
    lib = load_event_ref()
    assert lib is not None, "oracle/_ref/libeventdrv.so is not built (make -C oracle all && make -C oracle -f event.mk)"
    trials = []
    for i, (r, keys, times) in enumerate(ref_run(lib, MASTER, 0, TRIALS)):
        assert r.events < TRACE_CAP
        trials.append({"seed": fmix64(MASTER, i), "events": r.events, "t_end": float(r.t_end).hex(), "counters": list(r.counter),
                       "trace": [[k, float(t).hex()] for k, t in zip(keys, times)]})
    lines = ",\n".join(json.dumps(t, separators=(",", ":")) for t in trials)       # one trial per line
    VECTORS.write_text('{"master": %d, "trials": [\n%s\n]}\n' % (MASTER, lines))
    print(TRIALS, "trials, events", min(t["events"] for t in trials), "..", max(t["events"] for t in trials))


if __name__ == "__main__":
    main()
