#!/usr/bin/env python3
"""A/B of two builds of the C-ABI library on bench.py's headline workload (run on a GPU machine):

    python scripts/build_variant.py parent            # from a checkout of the baseline commit (nvcc, no GPU needed)
    python scripts/mm1_ab.py cimba_b200/lib/variants/parent.so cimba_b200/lib/libcimba_b200.so --reps 3

Prints the card's name, power limit and SM clock, then runs `bench.py --gpus 1 --steps 5 --warmup 3 --no-cpu-baseline --no-e2e
--no-secondary` (or --bench-args) REPS times per build, alternating A and B, with CIMBA_B200_LIB selecting the build.  One JSON
line per run, then a summary: the median events/s of each build, B's gain over A, and whether every B run beat every A run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def bench(lib, args):
    env = dict(os.environ, CIMBA_B200_LIB=str(Path(lib).resolve()))
    p = subprocess.run([sys.executable, str(ROOT / "bench.py"), *args], capture_output=True, text=True, env=env, cwd=ROOT)
    if p.returncode != 0:
        sys.exit(f"bench.py failed with {lib}:\n{p.stderr[-4000:]}")
    lines = [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")]
    return [l for l in lines if "metric" in l][-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a", help="library A (the baseline)")
    ap.add_argument("b", help="library B")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--bench-args", default="--gpus 1 --steps 5 --warmup 3 --no-cpu-baseline --no-e2e --no-secondary")
    o = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    runs = {"a": [], "b": []}
    for rep in range(o.reps):
        for tag, lib in (("a", o.a), ("b", o.b)):
            r = bench(lib, o.bench_args.split())
            runs[tag].append(r["value"])
            print(json.dumps({"run": rep, "lib": tag, "path": lib, "events_per_s": r["value"],
                              "result": {k: v for k, v in r.items() if not isinstance(v, (dict, list))}}), flush=True)
    ma, mb = statistics.median(runs["a"]), statistics.median(runs["b"])
    print(json.dumps({"median_a": ma, "median_b": mb, "gain_b_over_a": mb / ma - 1.0,
                      "every_b_beats_every_a": min(runs["b"]) > max(runs["a"])}), flush=True)


if __name__ == "__main__":
    main()
