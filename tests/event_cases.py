"""Shared by tests/test_event_queue.py, tests/test_gpu_event_queue.py and tests/golden/make_event_golden.py: the trial seeds of
examples/event_model.cuh's EventTestT, the oracles of the reference's event-queue test (oracle/event.mk: the unmodified program
oracle/_ref/test_event and oracle/ref_build/event_driver.c in oracle/_ref/libeventdrv.so) and the stored vectors.

Trial i is seeded fmix64(MASTER, i) (cmb_random_fmix64, src/cmb_random.c:70-80).  MASTER is chosen so that trial 0's seed is
GOLDEN_SEED, the seed of the reference's golden file test/reference/event.txt (tests/golden/event.txt): fmix64 is a bijection,
and MASTER is its inverse at that seed."""
import ctypes as C
import json
from pathlib import Path

from oracle_libs import Result

ROOT = Path(__file__).resolve().parents[1]
M64 = (1 << 64) - 1
GOLDEN_SEED = 0x34F05C64D7AD598F
VECTORS = ROOT / "tests/golden/event_vectors.json"
TRACE_CAP = 256             # more pops than any EventTestT trial has (about 60)


def fmix64(seed, nonce):
    h = (seed + nonce) & M64
    h ^= h >> 33
    h = (h * 0xFF51AFD7ED558CCD) & M64
    h ^= h >> 33
    h = (h * 0xC4CEB9FE1A85EC53) & M64
    h ^= h >> 33
    return h


def fmix64_inverse(h):
    """The x with fmix64(x, 0) == h (x ^= x >> 33 is its own inverse on 64 bits)."""
    h ^= h >> 33
    h = (h * pow(0xC4CEB9FE1A85EC53, -1, 1 << 64)) & M64
    h ^= h >> 33
    h = (h * pow(0xFF51AFD7ED558CCD, -1, 1 << 64)) & M64
    h ^= h >> 33
    return h


MASTER = fmix64_inverse(GOLDEN_SEED)
assert fmix64(MASTER, 0) == GOLDEN_SEED


def load_event_ref():
    """oracle/_ref/libeventdrv.so, or None where it was not built (the reference sources are absent)."""
    so = ROOT / "oracle/_ref/libeventdrv.so"
    if not so.exists():
        return None
    lib = C.CDLL(str(so))
    lib.event_ref_run_trials.restype = C.c_int
    lib.event_ref_run_trials.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64),
                                         C.POINTER(C.c_double), C.POINTER(Result)]
    return lib


def ref_run(lib, master, first, count, cap=TRACE_CAP):
    """[(result, keys, times)] of trials [first, first + count), the pop trace cut at the events executed."""
    out = (Result * count)()
    keys = (C.c_uint64 * (count * cap))()
    times = (C.c_double * (count * cap))()
    assert lib.event_ref_run_trials(master, first, count, cap, keys, times, out) == 0
    res = []
    for i, r in enumerate(out):
        n = min(r.events, cap)
        res.append((r, list(keys[i * cap:i * cap + n]), list(times[i * cap:i * cap + n])))
    return res


def vectors():
    return json.loads(VECTORS.read_text())
