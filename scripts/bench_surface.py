"""Events per second of the walk-in clinic (examples/clinic_model.cuh: every cmb_random distribution model code has, alias
routing, summaries) on the static tier and on the general engine, both as user-built model libraries.

    python scripts/bench_surface.py [--trials 65536] [--groups 2000] [--general-groups 2000] [--reps 3] [--out F]

* the card's name, power limit and SM clock, read with one nvidia-smi call before the runs;
* the static library (examples/clinic_static_user_model.cu) at `trials` x `groups` arrival groups;
* the general-engine library (examples/clinic_user_model.cu) on the same trials at `general_groups` groups;
* events/s of each: one warm-up launch, then `reps` timed launches (CUDA events), best and median; the static library's
  hand-overs to the general engine (diag[2]) are reported;
* 16 trials of both libraries at `general_groups` groups, bit for bit (events, patients, clock, time in clinic, counters).

Arrival groups every 2.0 on average, service scale 0.6 (the desks' loads 0.4-0.6); queues spill past 32 entries into 4096 per
queue.  Prints one JSON line; --out writes it to a file as well."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
import build_model                  # noqa: E402
import cimba_b200 as cb             # noqa: E402

MASTER = 0x34F05C64D7AD598F
ARR, SRV, SPILL = 2.0, 0.6, 4096


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power, sm, sm_max = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def launch(mid, n, groups, first=0):
    dev = torch.device("cuda", torch.cuda.current_device())
    arr = torch.full((n,), ARR, dtype=torch.float64, device=dev)
    srv = torch.full((n,), SRV, dtype=torch.float64, device=dev)
    diag = torch.zeros(4, dtype=torch.int64, device=dev)
    res = cb.launch_trials(arr, srv, num_objects=groups, master_seed=MASTER, first_trial=first, model=mid,
                           queue_spill_cap=SPILL, params=[0], diag=diag)
    return res, diag


def rate(mid, n, groups, reps):
    launch(mid, n, groups)                              # warm-up: module load, workspace
    torch.cuda.synchronize()
    runs = []
    for _ in range(reps):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        res, diag = launch(mid, n, groups)
        t1.record()
        torch.cuda.synchronize()
        assert int(res.status.abs().sum().item()) == 0
        ev = int(res.events.sum().item())
        ms = t0.elapsed_time(t1)
        runs.append({"ms": round(ms, 2), "events": ev, "events_per_s": ev / (ms * 1e-3), "handed_on": int(diag[2].item())})
    r = sorted(x["events_per_s"] for x in runs)
    return {"trials": n, "groups": groups, "runs": runs, "best": r[-1], "median": r[len(r) // 2]}


def rows(res):
    return [(int(e), int(o), float(t).hex(), float(s).hex(), [int(v) for v in c])
            for e, o, t, s, c in zip(res.events.cpu().tolist(), res.objects.cpu().tolist(), res.t_end.cpu().tolist(),
                                     res.sum_wait.cpu().tolist(), res.counters.cpu().numpy().astype(np.uint64))]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--trials", type=int, default=65536)
    ap.add_argument("--groups", type=int, default=2000)
    ap.add_argument("--general-groups", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    info = card()
    static = cb.load_model(build_model.build(ROOT / "examples/clinic_static_user_model.cu"))
    general = cb.load_model(build_model.build(ROOT / "examples/clinic_user_model.cu"))
    out = {"card": info, "model": "clinic (examples/clinic_model.cuh)", "arr_mean": ARR, "srv_mean": SRV, "queue_spill_cap": SPILL,
           "static": rate(static, a.trials, a.groups, a.reps), "general": rate(general, a.trials, a.general_groups, a.reps)}
    s, g = launch(static, 16, a.general_groups, first=7)[0], launch(general, 16, a.general_groups, first=7)[0]
    torch.cuda.synchronize()
    out["sample_16_bit_identical"] = rows(s) == rows(g)
    out["speedup_median"] = out["static"]["median"] / out["general"]["median"]
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    assert out["sample_16_bit_identical"]


if __name__ == "__main__":
    main()
