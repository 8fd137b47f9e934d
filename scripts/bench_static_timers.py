"""Events per second of model 8 (FrontDeskT: timers, yield + resume, waits on a process and on events, a condition observing the
desk's guard, under interrupts) on three routes of the library: the default timers_kernel with its repair pass (variant 0), the
static tier (CIMBA_B200_VARIANT_STATIC) and the general engine (CIMBA_B200_VARIANT_GENERAL).

    python scripts/bench_static_timers.py [--trials 506880] [--general-trials N] [--duration 500]
                                          [--engines default,static,general] [--reps 3] [--warmup 64] [--sample 4096] [--out F]

* the card's name, power limit and SM clock, read with one nvidia-smi call before the runs;
* the inputs, results and workspace of each route allocated first (outside the timed window); one warm-up launch of each route
  (`warmup` trials: module load, stack limit); then `reps` rounds of one launch per route, in turn, CUDA events around the library
  call alone; the median events/s of each route and the ratios.  Each launch's time goes to stderr as it ends;
* the last timed launch of each route compared bit for bit over a sample of trials spread across the launch (events, objects,
  clock, sums, fel_high, counters), a SHA-256 of those rows, and diag[2] of the static route (trials its repair pass re-ran).

Sizes (H100, 132 SMs): all three routes launch 64-lane CTAs.  The general engine runs at most 4 of them per SM - 33 792 lanes - and
takes further trials grid-stride; timers_kernel and the static tier launch one lane per trial.  The default 506 880 = 132 x 64 x 60
trials is a whole number of waves for any count of CTAs per SM that divides 60, and a multiple of 33 792.  500 time units per
trial at means 1.0: about 5 400 events per trial.  Prints one JSON line; --out writes it to a file as well."""
import argparse
import hashlib
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import cimba_b200 as cb             # noqa: E402

MASTER = 0x34F05C64D7AD598F
VARIANT = {"default": 0, "static": cb.VARIANT_STATIC, "general": cb.VARIANT_GENERAL}


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power, sm, sm_max = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


class Launch:
    """One route's launch of `n` trials of model 8, everything it needs allocated up front."""

    def __init__(self, n, engine, duration):
        self.n, self.engine, self.variant, self.nobj = n, engine, VARIANT[engine], duration
        dev = torch.device("cuda", torch.cuda.current_device())
        self.ones = torch.ones(n, dtype=torch.float64, device=dev)
        self.diag = torch.zeros(4, dtype=torch.int64, device=dev)
        self.buffers = cb.TrialBuffers(n, dev, 0, cb.MODEL_TIMERS, 1, self.variant, 0, self.nobj)

    def run(self):
        self.diag.zero_()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        res = cb.launch_trials(self.ones, self.ones, num_objects=self.nobj, master_seed=MASTER, model=cb.MODEL_TIMERS, servers=1,
                               variant=self.variant, buffers=self.buffers, diag=self.diag)
        t1.record()
        torch.cuda.synchronize()
        assert int(res.status.abs().sum().item()) == 0, self.engine
        ev = int(res.events.sum().item())
        ms = t0.elapsed_time(t1)
        print(f"model 8 {self.engine}: {self.n} trials, {ev} events, {ms:.1f} ms", file=sys.stderr, flush=True)
        return res, int(self.diag[2].item()), {"ms": round(ms, 1), "events": ev, "events_per_s": ev / (ms * 1e-3)}


def rows(res, idx):
    t = torch.as_tensor(idx, device=res.events.device)
    cnt = np.ascontiguousarray(res.counters[t].cpu().numpy(), dtype=np.int64).view(np.uint64)
    return [(int(e), int(o), float(te).hex(), float(s).hex(), int(q), [int(v) for v in c])
            for e, o, te, s, q, c in zip(res.events[t].cpu().tolist(), res.objects[t].cpu().tolist(), res.t_end[t].cpu().tolist(),
                                         res.sum_wait[t].cpu().tolist(), res.max_queue[t].cpu().tolist(), cnt)]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--trials", type=int, default=506880)
    ap.add_argument("--general-trials", type=int, default=0, help="trials of the general engine's launches (0 = --trials)")
    ap.add_argument("--duration", type=int, default=500, help="time units per trial")
    ap.add_argument("--engines", default="default,static,general")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=64, help="trials of the warm-up launch of each route (0 = none)")
    ap.add_argument("--sample", type=int, default=4096, help="trials compared bit for bit across the routes")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    engines = [e for e in a.engines.split(",") if e]
    assert engines and all(e in VARIANT for e in engines), a.engines
    trials = {"default": a.trials, "static": a.trials, "general": a.general_trials or a.trials}
    out = {"card": card(), "model": 8, "duration": a.duration, "trials": {e: trials[e] for e in engines}}
    if a.warmup > 0:
        for e in engines:
            Launch(a.warmup, e, a.duration).run()
    launches = {e: Launch(trials[e], e, a.duration) for e in engines}
    runs = {e: [] for e in engines}
    last = {}
    for _ in range(a.reps):
        for e in engines:
            res, repaired, r = launches[e].run()
            runs[e].append(r)
            last[e] = (res, repaired)
    k = min(trials[e] for e in engines)                 # the trials every route ran
    idx = np.unique(np.linspace(0, k - 1, min(a.sample, k)).astype(np.int64))
    got = {e: rows(last[e][0], idx) for e in engines}
    out["runs"] = runs
    out["compared_trials"] = int(len(idx))
    out["rows_sha256"] = {e: hashlib.sha256(repr(got[e]).encode()).hexdigest() for e in engines}
    for e in engines:
        out[f"{e}_median"] = sorted(x["events_per_s"] for x in runs[e])[len(runs[e]) // 2]
    if "static" in engines:
        out["static_repaired"] = last["static"][1]
        for e in ("default", "general"):
            if e in engines:
                out[f"static_over_{e}"] = out["static_median"] / out[f"{e}_median"]
    out["bit_identical"] = all(got[e] == got[engines[0]] for e in engines)
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    assert out["bit_identical"], "the routes disagree"


if __name__ == "__main__":
    main()
