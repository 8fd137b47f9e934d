"""cimba_b200 - H100-native replication-parallel discrete-event engine.

Host-side mirror of the reference's experiment interface (ambonvik/cimba,
include/cimba.h) over the C-ABI library in include/cimba_b200.h.  PyTorch is
used for device memory, streams and torch.distributed only; all simulation work
happens in the hand-written sm_90a kernels under cimba_b200/csrc.
"""
from ._lib import (MODEL_MM1, MODEL_GG1, MODEL_MMC, MODEL_GUARDED, MODEL_PREEMPT, MODEL_BUFFER, MODEL_PRIOQ, MODEL_HOLD, MODEL_TIMERS, MODEL_MM1_RECORDED, MODEL_HARBOR, MODEL_GUARDED_RECORDED, MODEL_BUFFER_RECORDED, MODEL_PRIOQ_RECORDED, MODEL_RESOURCE_RECORDED, MODEL_AWACS, MODEL_RENEGE, MODEL_POOL_RECORDED, MODEL_TUTORIAL1, MODEL_PARK, MODEL_TUTORIAL2, MODEL_USER_BASE, VARIANT_GENERAL, VARIANT_STATIC, MAP_LANE, MAP_WARP, CimbaError, lib,
                   TRIAL_QUEUE_OVERFLOW, TRIAL_FEL_OVERFLOW, TRIAL_KEY_OVERFLOW, TRIAL_GUARD_OVERFLOW, TRIAL_PROC_OVERFLOW,
                   TRIAL_NEGATIVE_HOLD, TRIAL_ARENA_EXHAUSTED, TRIAL_BAD_ARGUMENT)
from .experiment import (TrialResults, TrialBuffers, cimba_run_experiment, launch_trials, run_trials, load_model,
                         rng_draws, rng_draws_ex, alias_create, fmix64, TRIAL_DTYPE,
                         awacs_set_terrain, awacs_upload_terrain, awacs_run)
from .summary import (DataSummary, WtdSummary, summarize_on_device, merge_across_ranks,
                      summarize_weighted_on_device, merge_weighted_rows_on_device, merge_weighted_across_ranks)

__all__ = [
    "MODEL_MM1", "MODEL_GG1", "MODEL_MMC", "MODEL_GUARDED", "MODEL_PREEMPT", "MODEL_BUFFER", "MODEL_PRIOQ", "MODEL_HOLD", "MODEL_TIMERS", "MODEL_MM1_RECORDED", "MODEL_HARBOR", "MODEL_GUARDED_RECORDED", "MODEL_BUFFER_RECORDED", "MODEL_PRIOQ_RECORDED", "MODEL_RESOURCE_RECORDED", "MODEL_AWACS", "MODEL_RENEGE", "MODEL_POOL_RECORDED", "MODEL_TUTORIAL1", "MODEL_PARK", "MODEL_TUTORIAL2", "MODEL_USER_BASE", "VARIANT_GENERAL", "VARIANT_STATIC", "load_model", "TrialBuffers", "awacs_set_terrain", "awacs_upload_terrain", "awacs_run", "MAP_LANE", "MAP_WARP", "CimbaError", "lib",
    "TRIAL_QUEUE_OVERFLOW", "TRIAL_FEL_OVERFLOW", "TRIAL_KEY_OVERFLOW", "TRIAL_GUARD_OVERFLOW", "TRIAL_PROC_OVERFLOW", "TRIAL_NEGATIVE_HOLD",
    "TRIAL_ARENA_EXHAUSTED", "TRIAL_BAD_ARGUMENT",
    "TrialResults", "cimba_run_experiment", "launch_trials", "run_trials", "rng_draws", "rng_draws_ex", "alias_create", "fmix64",
    "TRIAL_DTYPE", "DataSummary", "WtdSummary", "summarize_on_device", "merge_across_ranks",
    "summarize_weighted_on_device", "merge_weighted_rows_on_device", "merge_weighted_across_ranks",
]
__version__ = lib.cimba_b200_version().decode()
