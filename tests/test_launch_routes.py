"""cimba_b200_workspace_bytes (no device needed) over a grid of jobs: every built-in model id and an unloaded user id, odd
variants and server counts, two trial counts, the default, a large and an invalid spill cap.  Which route serves a job decides
the bytes, so a routing change that sends any of these jobs elsewhere, or changes an arena formula, fails here.

The expected values were recorded from the library as it was before its routes were gathered into one table
(record_workspace_bytes below)."""
import ctypes as C
import itertools
import json
import sys
from pathlib import Path

FIXTURE = Path(__file__).resolve().parent / "golden" / "launch_routes_workspace.json"
GRID = {
    "model": list(range(23)) + [1000 + 4095],       # CIMBA_B200_MODEL_USER_BASE + an id nobody loads
    "variant": [0, 1, 2, 3, 4, 16, 17, 99],
    "servers": [0, 1, 14, 15, 16, 17, 64, 1081, 40000],
    "num_trials": [1, 4097],
    "queue_spill_cap": [0, 8192, 3],
}


def workspace_bytes(lib, device_job):
    """Every grid point's cimba_b200_workspace_bytes from the library `lib`, in itertools.product order of GRID."""
    fn = lib.cimba_b200_workspace_bytes
    fn.restype, fn.argtypes = C.c_uint64, [C.c_void_p]
    out = []
    for point in itertools.product(*GRID.values()):
        job = device_job(**dict(zip(GRID, point)))
        out.append(int(fn(C.byref(job))))
    return out


def record_workspace_bytes(lib_path):
    """Rewrite the fixture from the library at lib_path: python tests/test_launch_routes.py --record path/to/libcimba_b200.so"""
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    from cimba_b200._lib import DeviceJob
    FIXTURE.write_text(json.dumps({"grid": GRID, "bytes": workspace_bytes(C.CDLL(str(lib_path)), DeviceJob)}) + "\n")


def test_workspace_bytes_of_every_route_are_unchanged(cb):
    from cimba_b200 import _lib
    want = json.loads(FIXTURE.read_text())
    assert want["grid"] == GRID
    got = workspace_bytes(_lib.lib, _lib.DeviceJob)
    points = list(itertools.product(*GRID.values()))
    assert len(got) == len(want["bytes"]) == len(points) == 24 * 8 * 9 * 2 * 3
    bad = [(dict(zip(GRID, p)), w, g) for p, w, g in zip(points, want["bytes"], got) if w != g]
    assert not bad, f"{len(bad)} jobs changed (job, recorded, now): {bad[:8]}"
    assert len(set(want["bytes"])) > 40                 # the grid reaches many routes, not one formula


if __name__ == "__main__":
    if sys.argv[1:2] != ["--record"] or len(sys.argv) != 3:
        sys.exit(record_workspace_bytes.__doc__)
    record_workspace_bytes(sys.argv[2])
