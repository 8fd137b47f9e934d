"""Shared by tests/test_growth_arena.py (CPU) and tests/test_gpu_growth_arena.py (GPU): experiment-scale jobs whose repair pass or
general engine needs more growth arena than the workspace its route asks for (cimba_b200_workspace_bytes), and what their trials
need, as measured with the engine's host build (tests/cmb_engine_host.cpp).

A trial's need is the arena cursor when it ends: allocation order is fixed by the seed, so the trial runs unflagged exactly when
it finds that much arena.  The arena is shared by every trial of a launch and never reclaimed, so a launch needs the sum."""

MASTER = 0x5DEECE66D2B3F10B
SAMPLE = 64                     # trials per shape whose need the CPU measures; the sum is scaled to the shape's trial count

MM1_SHAPE = dict(trials=4096, num_objects=100_000, arr_mean=1 / 1.05, srv_mean=1.0, servers=1)
MMC_SHAPE = dict(trials=1024, num_objects=20_000, srv_mean=1.0)

# name: (library model id or example stem, host-build model, variant, servers, shape).  Default workspace routes:
# "fast" = a fixed-capacity kernel with HBM rings of queue_spill_cap (512) entries per trial, then the repair pass;
# "static" = the static tier's rings (one queue), then the repair pass; "engine" = the general engine alone, no rings.
GPU_SHAPES = {
    "mm1-v0":         (0, 0, 0, 1, "fast"),
    "mm1-v2":         (0, 0, 2, 1, "fast"),
    "mm1-static":     (0, 0, 17, 1, "static"),
    "mm1-general":    (0, 0, 16, 1, "engine"),
    "gg1-v0":         (1, 1, 0, 1, "fast"),
    "gg1-static":     (1, 1, 17, 1, "static"),
    "gg1-general":    (1, 1, 16, 1, "engine"),
    "mm1rec-v0":      (9, 9, 0, 1, "fast"),
    "mm1rec-static":  (9, 9, 17, 1, "static"),
    "mm1rec-general": (9, 9, 16, 1, "engine"),
    "mmc8-fast":      (2, 2, 0, 8, "fast"),
    "mmc20-engine":   (2, 2, 0, 20, "engine"),
    "user-mm1":       ("mm1_user_model", 0, 0, 1, "engine"),
    "user-mm1-static": ("mm1_static_user_model", 0, 0, 1, "static"),
}

# The summed need of SAMPLE strided trials (sample_trials below) of each shape, in bytes, from the host build
# (tests/test_growth_arena.py checks these figures).  Per trial: M/M/1, G/G/1 and recorded M/M/1 at rho = 1.05 with 10^5 objects
# about 128 KB (the object queue's ring doubles to 8 192 entries, and the blocks it leaves behind stay allocated); M/M/c at
# rho = 1.25 with 2 * 10^4 objects 1.3 to 2.7 MB (a customer process per arrival and the guard's heap).
SAMPLED_NEED = {
    "mm1": 8_118_272,           # 65 408 .. 130 944 per trial: ~496 MB for 4096 trials
    "gg1": 8_380_416,           # 130 944 per trial: ~512 MB
    "mm1rec": 8_118_272,        # as M/M/1: ~496 MB
    "mmc8": 112_850_784,        # 1 376 208 .. 2 752 512 per trial: ~1.7 GB for 1024 trials
    "mmc20": 118_275_008,       # 1 381 088 .. 2 757 392 per trial: ~1.8 GB
}


def need_key(name):
    """The SAMPLED_NEED entry of a GPU shape: the shapes of one model and server count share their trials' needs."""
    stem = name.split("-")[0]
    return "mm1" if stem == "user" else stem


def shape_of(name):
    """(host-build model, servers, trials, num_objects, arr_mean, srv_mean) of a GPU shape"""
    _, host_model, _, servers, _ = GPU_SHAPES[name]
    if host_model == 2:
        return host_model, servers, MMC_SHAPE["trials"], MMC_SHAPE["num_objects"], 1.0 / (servers * 1.25), MMC_SHAPE["srv_mean"]
    return host_model, servers, MM1_SHAPE["trials"], MM1_SHAPE["num_objects"], MM1_SHAPE["arr_mean"], MM1_SHAPE["srv_mean"]


def sample_trials(trials):
    return [i * trials // SAMPLE for i in range(SAMPLE)]


def estimated_need(name):
    """The summed need of all the shape's trials, scaled from the sample"""
    trials = shape_of(name)[2]
    return SAMPLED_NEED[need_key(name)] * trials // SAMPLE


def rings_bytes(name, trials, spill_cap=512):
    """The bytes in front of the growth arena in the workspace of the shape's default route"""
    kind = GPU_SHAPES[name][4]
    return 0 if kind == "engine" else (trials * spill_cap * 8 + 255) // 256 * 256
