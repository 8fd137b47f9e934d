#!/usr/bin/env python3
"""Cost of one warp event step of mm1_kernel at several loads, for one or more builds of the C-ABI library (run on a GPU
machine):

    python scripts/build_variant.py parent            # from a checkout of the baseline commit (nvcc, no GPU needed)
    python scripts/mm1_window_cost.py cimba_b200/lib/variants/parent.so cimba_b200/lib/libcimba_b200.so --reps 3

Each build runs in a process of its own (CIMBA_B200_LIB selects it), REPS times, the builds alternating.  A run launches
--trials M/M/1 trials x --objects objects at every rho of --rhos (service mean 1, arrival mean 1 / rho), one warm-up
launch and --launches timed ones per rho, and reports the time per warp event step: CUDA-event time of the launch over
the mean event steps per warp the kernel itself counted (diag[0] / diag[1]).  The launch includes the repair pass, which
re-runs the trials whose queue outgrew the on-chip window plus the spill ring (none at these sizes with the default ring).

Prints the card's name, power limit and SM clock, one JSON line per run, then per build and rho the median ns per warp
step and its ratio to the rho = 0.8 row of the same build."""
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
MASTER_SEED = 0x34F05C64D7AD598F


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def worker(o):
    sys.path.insert(0, str(ROOT))
    import torch
    import cimba_b200 as cb
    from cimba_b200.experiment import TrialBuffers

    assert torch.cuda.is_available(), "mm1_window_cost.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bufs = TrialBuffers(o.trials, dev, 0, cb.MODEL_MM1, 1, 0)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    srv = torch.ones(o.trials, dtype=torch.float64, device=dev)
    rows = {}
    for rho in o.rhos:
        arr = torch.full((o.trials,), 1.0 / rho, dtype=torch.float64, device=dev)

        def launch():
            return cb.launch_trials(arr, srv, num_objects=o.objects, master_seed=MASTER_SEED, buffers=bufs, diag=diag)

        launch()
        torch.cuda.synchronize(dev)
        ns = []
        for _ in range(o.launches):
            diag.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = launch()
            e1.record()
            torch.cuda.synchronize(dev)
            d = diag.cpu().tolist()
            ns.append(e0.elapsed_time(e1) * 1e6 / (d[0] / d[1]))
        rows[str(rho)] = {"ns_per_warp_step": statistics.median(ns), "all": ns, "steps_per_warp": d[0] / d[1],
                          "events_per_trial": res.events.double().mean().item(),
                          "repaired": d[2], "failed": int((res.status != 0).sum().item())}
    print(json.dumps(rows), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+", help="builds of the library to compare")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trials", type=int, default=65536)
    ap.add_argument("--objects", type=int, default=100_000)
    ap.add_argument("--rhos", type=float, nargs="+", default=[0.5, 0.8, 0.9, 0.95])
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    o = ap.parse_args()
    if o.worker:
        worker(o)
        return
    print(json.dumps({"card": card()}), flush=True)
    runs = {lib: [] for lib in o.libs}
    args = ["--trials", str(o.trials), "--objects", str(o.objects), "--launches", str(o.launches),
            "--rhos", *map(str, o.rhos)]
    for rep in range(o.reps):
        for lib in o.libs:
            env = dict(os.environ, CIMBA_B200_LIB=str(Path(lib).resolve()))
            p = subprocess.run([sys.executable, __file__, lib, "--worker", *args], capture_output=True, text=True,
                               env=env, cwd=ROOT)
            if p.returncode != 0:
                sys.exit(f"run with {lib} failed:\n{p.stderr[-4000:]}")
            rows = json.loads([l for l in p.stdout.splitlines() if l.startswith("{")][-1])
            runs[lib].append(rows)
            print(json.dumps({"run": rep, "lib": lib, "rows": rows}), flush=True)
    print(json.dumps({"card": card()}), flush=True)
    for lib in o.libs:
        med = {rho: statistics.median(r[str(rho)]["ns_per_warp_step"] for r in runs[lib]) for rho in o.rhos}
        base = med.get(0.8)
        print(json.dumps({"lib": lib, "median_ns_per_warp_step": {str(k): round(v, 2) for k, v in med.items()},
                          "vs_rho_0.8": {str(k): round(v / base, 4) for k, v in med.items()} if base else None}),
              flush=True)
    if len(o.libs) > 1:
        a = o.libs[0]
        for lib in o.libs[1:]:
            print(json.dumps({"lib": lib, "vs": a, "ns_ratio": {
                str(rho): round(statistics.median(r[str(rho)]["ns_per_warp_step"] for r in runs[lib])
                                / statistics.median(r[str(rho)]["ns_per_warp_step"] for r in runs[a]), 4)
                for rho in o.rhos}}), flush=True)


if __name__ == "__main__":
    main()
