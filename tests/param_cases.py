"""Shared by tests/test_oracle_port.py (CPU) and tests/test_gpu_per_trial_parameters.py (GPU): a table of per-trial parameters
and the oracle run one trial at a time at each trial's own parameters.

cimba_run_experiment runs an array of trial structs, each with its own arr_mean and srv_mean (benchmark/MM1_multi.c:131-133;
tutorial 1 puts 39 utilisations into one array).  A kernel that reads another trial's parameters, or drops the service mean's
multiply on a rare path, passes any test whose trials share one parameter set with srv_mean = 1.0.  So here:

* every parameter cycles with a period coprime to 32 (7 for the load, 5 for the time scale), so every warp, every
  producer/consumer pair and every persistent warp's run of trials holds a mix of values;
* the time scales are not powers of two (1e-3 ... 1234.5), so a mean taken from the wrong trial changes the rounding of every
  clock value, and srv_mean is never 1.0, so dropping its multiply changes the answer;
* the queueing models (M/M/1, G/G/1, M/M/c, recorded M/M/1, the tandem library) mix trials whose queue stays in the 32-entry
  shared-memory window, trials that reach the HBM spill ring and trials that outgrow both (rho = 4): the last go to the repair pass;
* the time-bounded models (hold, harbor, the reference's test worlds 3-6, 8, 11-14, reneging, tutorial 1) keep their means near
  the ones the rest of the suite runs, so trial lengths stay bounded.
"""
import numpy as np

from oracle_libs import run_trials, trace_trial

MASTER = 0x5DEECE66D2B3F10B
FIRST = 4093                       # first_trial != 0: seeds follow the global trial index
N = 197                            # ragged: 6 full warps and 5 lanes of a seventh
TRACE_POPS = 2000

SCALES = (1e-3, 0.37, 3.7, 1234.5, 0.061)                  # period 5: the time unit of a queueing trial
RHO = (0.5, 0.9, 0.3, 1.3, 0.75, 0.6, 4.0)                 # period 7: window, window, window, spill ring, ..., beyond the ring
RHO_REPAIR = (0.5, 0.9, 0.3, 0.8, 0.75, 0.6, 4.0)          # every 7th trial overflows the fast kernels' tables, the rest do not
NEAR_ONE_A = (1.0, 0.5, 0.7, 0.3, 1.3, 0.37, 0.9)          # time-bounded models: means near the ones tested elsewhere
NEAR_ONE_S = (0.6, 0.93, 0.37, 1.2, 0.8)

# model -> (servers, num_objects, kind, model params).  `num_objects` is the object count of the queueing models and the
# duration of the time-bounded ones.  Models 4 and 14 take no means (the reference's test programs fix them); model 7 reads
# arr_mean only.
TABLE = {
    0:  (1, 1500, "queue", ()),
    1:  (1, 1500, "queue", ()),
    2:  (3, 1500, "pool", ()),
    9:  (1, 1500, "queue", ()),
    17: (4, 1500, "queue", ()),                             # the tandem library (examples/tandem_model.cuh)
    7:  (300, 10, "hold", ()),
    10: (6, 600, "harbor", ()),
    3:  (10, 300, "near", ()),
    4:  (20, 300, "near", ()),
    5:  (10, 300, "near", ()),
    6:  (8, 300, "near", ()),
    8:  (1, 300, "near", ()),
    11: (10, 300, "near", ()),
    12: (10, 300, "near", ()),
    13: (10, 300, "near", ()),
    14: (1, 300, "near", ()),
    16: (40, 300, "renege", (0.7,)),
    19: (1, 2000, "tutorial1", (100.0,)),
}


def per_trial_params(model, n=N, servers=None, rho=RHO):
    """(arr_mean[n], srv_mean[n]) for `model`: float64, all > 0, srv_mean never 1.0."""
    kind = TABLE[model][2]
    c = servers if servers is not None else TABLE[model][0]
    i = np.arange(n)
    if kind in ("queue", "pool"):
        srv = np.array([SCALES[k % 5] for k in i])
        load = np.array([rho[k % 7] for k in i])
        arr = srv / (load * (c if kind == "pool" else 1))
    elif kind == "hold":                                    # the mean of the workers' holds; srv_mean is not read
        arr = np.array([(0.5, 0.93, 2.0, 0.7, 1.3, 0.61, 1.7)[k % 7] for k in i])
        srv = np.array([NEAR_ONE_S[k % 5] for k in i])
    elif kind == "harbor":                                  # hours between ships, hours to unload a small ship
        arr = np.array([(2.0, 1.5, 2.5, 1.8, 1.45, 2.2, 1.6)[k % 7] for k in i])
        srv = np.array([(8.0, 10.0, 6.0, 9.0, 7.0)[k % 5] for k in i])
    elif kind == "renege":                                  # think time, service time
        arr = np.array([(3.0, 2.5, 3.7, 2.2, 3.3, 2.8, 4.1)[k % 7] for k in i])
        srv = np.array([(0.8, 1.1, 0.93, 1.2, 0.7)[k % 5] for k in i])
    elif kind == "tutorial1":
        srv = np.array([NEAR_ONE_S[k % 5] for k in i])
        arr = srv / np.array([(0.5, 0.9, 0.3, 0.8, 0.75, 0.6, 0.95)[k % 7] for k in i])
    else:
        arr = np.array([NEAR_ONE_A[k % 7] for k in i])
        srv = np.array([NEAR_ONE_S[k % 5] for k in i])
    arr, srv = arr.astype(np.float64), srv.astype(np.float64)
    assert (arr > 0).all() and (srv > 0).all() and not (srv == 1.0).any()
    return arr, srv


def oracle(lib, prefix, model, servers, nobj, arr, srv, master=MASTER, first=FIRST, par=0):
    """Trial i of the launch, run alone at its own parameters: seed fmix64(master, first + i)."""
    return [run_trials(lib, prefix, model, servers, master, first + i, 1, nobj, float(arr[i]), float(srv[i]), par)[0]
            for i in range(len(arr))]


def oracle_trace(lib, prefix, model, servers, nobj, arr, srv, i, fmix64, master=MASTER, first=FIRST, cap=TRACE_POPS):
    """(result, keys, times) of trial i's first `cap` pops."""
    return trace_trial(lib, prefix, model, servers, fmix64(master, first + i), nobj, float(arr[i]), float(srv[i]), cap)
