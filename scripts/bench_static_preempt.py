"""Events per second of the reference's fixed-process resource programs on the static tier (CIMBA_B200_VARIANT_STATIC) and on the
general engine (CIMBA_B200_VARIANT_GENERAL), through the library's built-in routes: tutorial/tut_2_1.c (model 21),
test/test_resourcepool.c (model 18) and test/test_resource.c (model 14).

    python scripts/bench_static_preempt.py [--models 18,14] [--trials 506880] [--general-trials N] [--engines static,general]
                                           [--reps 3] [--warmup 64] [--out F]

* the card's name, power limit and SM clock, read with one nvidia-smi call before the runs;
* per model: the inputs, results and workspace of each engine allocated first (outside the timed window); one warm-up launch of
  each engine (`warmup` trials: module load, stack limit); then `reps` rounds of one static and one general launch, alternating,
  CUDA events around the library call alone; the median events/s of each engine and their ratio.  Each launch's time goes to
  stderr as it ends;
* the last timed launch of each engine compared row for row over the trials both ran (events, objects, clock, sums, counters),
  a SHA-256 of those rows (to compare engines run in separate calls, `--engines`), and diag[2] == 0 (the tier answered every
  trial, not the repair pass behind it).

Sizes (H100, 132 SMs): the general engine launches at most CMB_RESIDENT_CTAS = 4 CTAs of 64 lanes per SM - 33 792 lanes - and
takes further trials grid-stride; the static tier launches one lane per trial, and fits 10 CTAs of 64 per SM for model 14
(80 registers and 20 KB of shared memory per CTA: 84 480 lanes) and 6 for models 18 and 21 (154 and 168 registers: 50 688
lanes).  The default 506 880 trials is a multiple of all three, so every engine runs full waves.  The pool test runs 20 units for
500 time units, the resource test 2 000.  Tutorial 2 has its own length (about 660 000 events per trial), so one of its launches
lasts as long as its slowest trial - minutes on the general engine; run it with --trials 50688 --general-trials 33792 (one full
wave of each engine) and, if need be, one engine per call (--engines).  Prints one JSON line; --out writes it to a file as well."""
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
SHAPE = {21: ("tutorial 2 (tutorial/tut_2_1.c)", 1, 0), 18: ("pool test (test/test_resourcepool.c)", 20, 500),
         14: ("resource test (test/test_resource.c)", 1, 2000)}
VARIANT = {"static": cb.VARIANT_STATIC, "general": cb.VARIANT_GENERAL}


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power, sm, sm_max = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


class Launch:
    """One engine's launch of `n` trials of `model`, everything it needs allocated up front."""

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
    k = min(trials.values())                            # the trials both engines run, whichever of them this call runs
    got = {e: rows(last[e][0], k) for e in engines}
    name, servers, nobj = SHAPE[model]
    out = {"model": model, "name": name, "servers": servers, "num_objects": nobj, "trials": {e: trials[e] for e in engines},
           "runs": runs, "compared_trials": k,
           "rows_sha256": {e: hashlib.sha256(repr(got[e]).encode()).hexdigest() for e in engines}}
    for e in engines:
        out[f"{e}_median"] = sorted(x["events_per_s"] for x in runs[e])[len(runs[e]) // 2]
    if "static" in engines:
        out["static_repaired"] = last["static"][1]
    if len(engines) == 2:
        out["static_over_general"] = out["static_median"] / out["general_median"]
        out["bit_identical"] = got["static"] == got["general"]
    del launches, last
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--models", default="18,14")
    ap.add_argument("--trials", type=int, default=506880)
    ap.add_argument("--general-trials", type=int, default=0, help="trials of the general engine's launches (0 = --trials)")
    ap.add_argument("--engines", default="static,general")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=64, help="trials of the warm-up launch of each engine (0 = none)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    engines = [e for e in a.engines.split(",") if e]
    assert engines and all(e in VARIANT for e in engines), a.engines
    trials = {"static": a.trials, "general": a.general_trials or a.trials}
    out = {"card": card(), "results": [bench(int(m), trials, engines, a.reps, a.warmup) for m in a.models.split(",")]}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    for r in out["results"]:
        assert r.get("bit_identical", True) and r.get("static_repaired", 0) == 0, r["model"]


if __name__ == "__main__":
    main()
