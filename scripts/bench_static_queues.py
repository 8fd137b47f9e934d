"""Events per second of the reference's queue and coverage programs on three routes of the library: the default fixed-capacity
kernel with its repair pass (variant 0), the static tier (CIMBA_B200_VARIANT_STATIC) and the general engine
(CIMBA_B200_VARIANT_GENERAL): test/test_objectqueue.c (models 3 and 11), test/test_priorityqueue.c (model 13), the
priority-queue-and-condition world of model 6, test/test_resourcepool.c's cast with checks (model 4, preempt_kernel by default)
and the buffer-and-resource world with test/test_buffer.c (models 5 and 12, buffer_kernel by default).

    python scripts/bench_static_queues.py [--models 3,11,13,6,4,5,12] [--trials 506880] [--general-trials N]
                                          [--engines default,static,general] [--reps 3] [--warmup 64] [--out F]

* the card's name, power limit and SM clock, read with one nvidia-smi call before the runs;
* per model: the inputs, results and workspace of each route allocated first (outside the timed window); one warm-up launch of
  each route (`warmup` trials: module load, stack limit); then `reps` rounds of one launch per route, in turn, CUDA events around
  the library call alone; the median events/s of each route and the ratios.  Each launch's time goes to stderr as it ends;
* the last timed launch of each route compared row for row over the trials all ran (events, objects, clock, sums, counters), a
  SHA-256 of those rows, and diag[2] of the static route (trials its repair pass re-ran: 0 when the tier answered them all).
  The run fails if the rows differ, or if the repair pass re-ran trials of a model the tier should answer alone at its shape -
  every model but 4, whose route keeps four spare event slots (the fewest its vector cases need) and leaves the trials that
  need a fifth, about 1.9 % at this shape, to the repair pass.

Sizes (H100, 132 SMs): all three routes launch 64-lane CTAs.  The general engine runs at most CMB_RESIDENT_CTAS = 4 of them per
SM - 33 792 lanes - and takes further trials grid-stride; the fixed-capacity kernel and the static tier launch one lane per trial,
as many CTAs per SM as their registers allow.  The default 506 880 = 132 x 64 x 60 trials is a whole number of waves for any
count of CTAs per SM that divides 60 (1-6, 10, 12, 15, 20), and a multiple of 33 792.  Capacity 10 and 500 time units per trial:
about 4 200 events per trial for the queue programs, 2 300 for model 4 and 4 500 / 5 800 for models 5 / 12.  Prints one JSON line; --out writes it to a file as well."""
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
# model -> (name, servers, num_objects)
SHAPE = {3: ("object queue test (test/test_objectqueue.c, no history)", 10, 500),
         11: ("object queue test (test/test_objectqueue.c)", 10, 500),
         13: ("priority queue test (test/test_priorityqueue.c)", 10, 500),
         6: ("priority queue + condition (model 6)", 10, 500),
         4: ("pool with priorities, pre-emption and interrupts (test/test_resourcepool.c's cast, model 4)", 10, 500),
         5: ("buffer + resource world (model 5)", 10, 500),
         12: ("buffer test (test/test_buffer.c)", 10, 500)}
REPAIRED_AT_SHAPE = {4}            # models whose static route leaves some trials of SHAPE to its repair pass (see above)
VARIANT = {"default": 0, "static": cb.VARIANT_STATIC, "general": cb.VARIANT_GENERAL}


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power, sm, sm_max = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


class Launch:
    """One route's launch of `n` trials of `model`, everything it needs allocated up front."""

    def __init__(self, model, n, engine):
        _, self.servers, self.nobj = SHAPE[model]
        self.model, self.n, self.engine, self.variant = model, n, engine, VARIANT[engine]
        dev = torch.device("cuda", torch.cuda.current_device())
        self.ones = torch.ones(n, dtype=torch.float64, device=dev)
        self.diag = torch.zeros(4, dtype=torch.int64, device=dev)
        self.buffers = cb.TrialBuffers(n, dev, 0, model, self.servers, self.variant, 0, self.nobj)

    def run(self):
        self.diag.zero_()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        res = cb.launch_trials(self.ones, self.ones, num_objects=self.nobj, master_seed=MASTER, model=self.model, servers=self.servers,
                               variant=self.variant, buffers=self.buffers, diag=self.diag)
        t1.record()
        torch.cuda.synchronize()
        assert int(res.status.abs().sum().item()) == 0, (self.model, self.engine)
        ev = int(res.events.sum().item())
        ms = t0.elapsed_time(t1)
        print(f"model {self.model} {self.engine}: {self.n} trials, {ev} events, {ms:.1f} ms", file=sys.stderr, flush=True)
        return res, int(self.diag[2].item()), {"ms": round(ms, 1), "events": ev, "events_per_s": ev / (ms * 1e-3)}


def rows(res, k):
    return [(int(e), int(o), float(t).hex(), float(s).hex(), [int(v) for v in c])
            for e, o, t, s, c in zip(res.events[:k].cpu().tolist(), res.objects[:k].cpu().tolist(), res.t_end[:k].cpu().tolist(),
                                     res.sum_wait[:k].cpu().tolist(), res.counters[:k].cpu().numpy().astype(np.uint64))]


def bench(model, trials, engines, reps, warmup):
    if warmup > 0:
        for engine in engines:
            Launch(model, warmup, engine).run()
    launches = {e: Launch(model, trials[e], e) for e in engines}
    runs = {e: [] for e in engines}
    last = {}
    for _ in range(reps):
        for e in engines:
            res, repaired, r = launches[e].run()
            runs[e].append(r)
            last[e] = (res, repaired)
    k = min(trials[e] for e in engines)                 # the trials every route of this call ran
    got = {e: rows(last[e][0], k) for e in engines}
    name, servers, nobj = SHAPE[model]
    out = {"model": model, "name": name, "servers": servers, "num_objects": nobj, "trials": {e: trials[e] for e in engines},
           "runs": runs, "compared_trials": k,
           "rows_sha256": {e: hashlib.sha256(repr(got[e]).encode()).hexdigest() for e in engines}}
    for e in engines:
        out[f"{e}_median"] = sorted(x["events_per_s"] for x in runs[e])[len(runs[e]) // 2]
    if "static" in engines:
        out["static_repaired"] = last["static"][1]
        for e in ("default", "general"):
            if e in engines:
                out[f"static_over_{e}"] = out["static_median"] / out[f"{e}_median"]
    out["bit_identical"] = all(got[e] == got[engines[0]] for e in engines)
    del launches, last
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--models", default="3,11,13,6")
    ap.add_argument("--trials", type=int, default=506880)
    ap.add_argument("--general-trials", type=int, default=0, help="trials of the general engine's launches (0 = --trials)")
    ap.add_argument("--engines", default="default,static,general")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=64, help="trials of the warm-up launch of each route (0 = none)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    engines = [e for e in a.engines.split(",") if e]
    assert engines and all(e in VARIANT for e in engines), a.engines
    trials = {"default": a.trials, "static": a.trials, "general": a.general_trials or a.trials}
    out = {"card": card(), "results": [bench(int(m), trials, engines, a.reps, a.warmup) for m in a.models.split(",")]}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    for r in out["results"]:
        assert r["bit_identical"] and (r.get("static_repaired", 0) == 0 or r["model"] in REPAIRED_AT_SHAPE), r["model"]


if __name__ == "__main__":
    main()
