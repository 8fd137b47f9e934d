"""Write tests/golden/random_sweep_vectors.json: every case of tests/random_sweep_cases.py drawn by the unmodified reference build
(oracle/_ref/librefdrv.so, ref_rng_draws_ex), N variates at seed cmb_random_fmix64(SEED, case index).

Per case: the SHA-256 of the variates' bit patterns (NaN written as one canonical NaN: CUDA's and x86's NaN payloads differ and a
NaN is a NaN); for the kinds whose variate is a libm result, the first 64 values; and from the host build of this project's
formulation (tests/random_sweep_host.cpp), the generator calls the stream made and the smallest margin of its Marsaglia-Tsang
log comparisons, which tests/test_gpu_random_sweep.py uses to decide which gamma-family cases may demand bit-exactness.

    make -C oracle ref && python tests/golden/make_random_sweep_golden.py"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "tests"))
import random_sweep_cases as rc          # noqa: E402
from oracle_libs import load_ref, rng_draws_ex      # noqa: E402
from random_sweep_cases import build_host, canonical, host_sweep, case_seed     # noqa: E402

OUT = ROOT / "tests/golden/random_sweep_vectors.json"
SPOT = 64


def main():
    ref = load_ref()
    if ref is None:
        sys.exit("oracle/_ref/librefdrv.so is not built (make -C oracle ref)")
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        host = build_host(Path(tmp))
        cases = []
        for i, ((kind, par), cid) in enumerate(zip(rc.CASES, rc.IDS)):
            seed = case_seed(i)
            v = np.array(rng_draws_ex(ref, "ref", seed, kind, par, rc.N))
            h = host_sweep(host, i)
            entry = {"id": cid, "kind": kind, "params": [float(x).hex() for x in par], "seed": seed, "n": rc.N,
                     "sha256": rc.stream_sha256(canonical(v)), "calls": h["calls"], "compares": h["compares"],
                     "margin": None if not np.isfinite(h["margin"]) else float(h["margin"])}
            if rc.libm_value(kind, par):
                entry["first"] = [float(x).hex() for x in v[:SPOT]]
            cases.append(entry)
    OUT.write_text(json.dumps({"seed": rc.SEED, "n": rc.N, "cases": cases}, indent=0) + "\n")
    print(f"wrote {OUT} ({len(cases)} cases)")


if __name__ == "__main__":
    main()
