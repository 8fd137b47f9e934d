/*
 * cimba_b200.h - C ABI of the H100-native replication-parallel discrete-event
 * engine.  Plain C, plain pointers and sizes; no CUDA or torch types.
 *
 * This is the GPU drop-in for the reference's experiment executive
 *
 *     void cimba_run_experiment(void *your_experiment_array,
 *                               uint64_t num_trials,
 *                               size_t trial_struct_size,
 *                               cimba_trial_func *your_trial_func);
 *                                   (reference include/cimba.h:144-147,
 *                                    src/cimba.c:151-188)
 *
 * A C function pointer cannot run on the device, so `your_trial_func` is
 * replaced by a model descriptor naming one of the device-resident models and
 * telling the library where the parameter and result fields sit inside the
 * caller's trial struct.  Everything else keeps the reference's contract: the
 * caller owns the array, the call blocks until every trial has run, results are
 * written in place, trials are independent, and trial i is seeded with
 * cmb_random_fmix64(master_seed, first_trial + i) (src/cmb_random.c:70-80, the
 * scheme of test/test_cimba.c:396).
 *
 * Errors: the reference has no error codes (violations abort through
 * cmb_assert_release -> cmi_assert_failed, include/cmb_assert.h:44-80).  Here
 * every entry point returns 0 on success or a negative CIMBA_B200_E* code and
 * never aborts the host process; per-trial capacity violations come back in the
 * per-trial status word.  There is NO CPU fallback: without a CUDA device the
 * calls fail with CIMBA_B200_ENODEVICE.
 */
#ifndef CIMBA_B200_H
#define CIMBA_B200_H

#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CIMBA_B200_VERSION_STRING "0.1.0"

/* Device-resident models (SURVEY.md section 8d workloads). */
#define CIMBA_B200_MODEL_MM1 0   /* benchmark/MM1_multi.c:52-89: exp arrivals, exp service, cmb_objectqueue */
#define CIMBA_B200_MODEL_GG1 1   /* same structure: cmb_random_erlang(2, m/2) arrivals, normal(m, m/4) service redrawn while < 0 */
#define CIMBA_B200_MODEL_MMC 2   /* generator + one process per customer contending for a cmb_resourcepool of `servers` units */
#define CIMBA_B200_MODEL_GUARDED 3 /* test/test_objectqueue.c: 3 putters + 3 getters with random priorities on a BOUNDED
                                    * cmb_objectqueue (capacity = `servers` <= 16), a nuisance process interrupting them,
                                    * an end event at t = num_objects stopping everybody (general cancel/interrupt path) */
#define CIMBA_B200_MODEL_PREEMPT 4 /* test/test_resourcepool.c: 3 mice (priority_set + acquire), 2 rats (pre-empt), a cat
                                    * interrupting them, on a cmb_resourcepool of `servers` units; end event at t = num_objects */
#define CIMBA_B200_MODEL_BUFFER 5  /* test/test_buffer.c + test/test_resource.c: 2 fillers + 2 drainers on a cmb_buffer of capacity
                                    * `servers`, a polite and a pre-empting worker on one cmb_resource, a nuisance; end at t = num_objects */
#define CIMBA_B200_MODEL_HOLD 7    /* the hold model: `servers` <= 33 822 processes in cmb_process_hold(exp(arr_mean)) loops + a 1.0 s
                                    * ticker + an end event at t = num_objects (tutorial/tut_5_1.c's event-list shape); one trial
                                    * per WARP, 32-ary heap: root + level 1 in registers, deeper levels in HBM/L2 moved as coalesced
                                    * 512-byte rows (variant 1: the whole list in shared memory, <= 1080 processes) */
#define CIMBA_B200_MODEL_PRIOQ 6   /* test/test_priorityqueue.c + test/test_condition.c: 2 producers, a consumer and a shuffler
                                    * (position / reprioritize / cancel by handle) on a cmb_priorityqueue of capacity `servers` <= 15,
                                    * a tide process signalling a cmb_condition two waiters watch, a nuisance; end at t = num_objects */
#define CIMBA_B200_MODEL_TIMERS 8   /* tutorial/tut_3_1.c + test/test_process.c + test/test_event.c: two patients reneging on a
                                    * cmb_resource with cmb_process_timer_add / timer_cancel / timers_clear / timer_set + yield,
                                    * a clerk (cmb_process_resume, cmb_process_exit), a supervisor (cmb_process_wait_process, restart),
                                    * a ringer (cmb_event_reschedule / reprioritize / cancel, cmb_process_wait_event), a listener,
                                    * a watcher on a condition OBSERVING the desk's guard, a nuisance; end at t = num_objects */
#define CIMBA_B200_MODEL_MM1_RECORDED 9 /* MODEL_MM1 with the queue's history on (cmb_objectqueue_recording_start, as
                                    * tutorial/tut_1_*.c and test/test_cimba.c run it): counters[trial][0..7] receive the
                                    * time-weighted queue-length cmb_wtdsummary {count, min, max, m1, m2, m3, m4, wsum}
                                    * (count as u64, the rest as IEEE-754 bit patterns) that cmb_timeseries_summarize
                                    * (src/cmb_timeseries.c:167-188) computes from the stored history - folded on the fly */
#define CIMBA_B200_MODEL_HARBOR 10   /* test/test_condition.c (= tutorial/tut_4_1.c), the reference's harbor: weather and tide processes
                                    * signalling a cmb_condition every hour, one ship PROCESS per arrival (up to 120 alive at once)
                                    * waiting on it with a predicate over depth, wind, `servers` tugs and 6 + 3 berths held in three
                                    * cmb_resourcepools, a departure process on a second condition, an end event at t = num_objects
                                    * hours.  arr_mean = mean inter-arrival time, srv_mean = mean unloading time of a small ship.
                                    * counters: ships through (small, large), their mean system times, tug / berth history summaries,
                                    * harbormaster reactivations - with the golden seed and 873 600 h exactly test/reference/condition.txt.
                                    * variant 0: up to 32 768 trials run one per WARP with the state in shared memory (tables for 43 ships
                                    * alive) and any trial that outgrows them is re-run one per lane with the HBM tables (120 ships);
                                    * 1 = warp-per-trial only, 2 = lane-per-trial only */
#define CIMBA_B200_MODEL_GUARDED_RECORDED 11 /* MODEL_GUARDED with the queue's history on = test/test_objectqueue.c as it stands:
                                    * counters[6] = time-weighted mean queue length (bits), max_queue = history samples with a
                                    * duration; capacity 10, means 1, 1e6 time units and the golden seed give
                                    * test/reference/objectqueue.txt's "N 5689021  Mean 5.008" */
#define CIMBA_B200_MODEL_BUFFER_RECORDED 12 /* test/test_buffer.c as it stands: three putters and three getters moving 1..15 units
                                    * through a cmb_buffer of capacity `servers`, a nuisance, the level history on.  counters[4] =
                                    * time-weighted mean level (bits), max_queue = history samples with a duration; capacity 10, means 1,
                                    * 10 000 time units and the golden seed give test/reference/buffer.txt's "N 41876  Mean 4.980" */
#define CIMBA_B200_MODEL_PRIOQ_RECORDED 13 /* test/test_priorityqueue.c: MODEL_GUARDED_RECORDED's seven processes on a cmb_priorityqueue
                                    * (capacity `servers` <= 15), objects put with the putter's own priority; same outputs.  Capacity 10,
                                    * means 1, 1e6 time units and the golden seed give test/reference/priorityqueue.txt's
                                    * "N 5689021  Mean 5.008" */
#define CIMBA_B200_MODEL_RESOURCE_RECORDED 14 /* test/test_resource.c as it stands: three pre-emptable processes and a pre-empter on one
                                    * cmb_resource, usage history on.  counters: [0] acquisitions by the targets [1] PREEMPTED received
                                    * [2] acquisitions by the pre-empter [3] time-weighted mean utilisation (bits) [4] time of the first
                                    * pre-emption (bits) [5] its victim + 1; max_queue = history samples.  25 time units and the golden
                                    * seed give test/reference/resource.txt: "N 30  Mean 0.9816", Target_3 pre-empted at t = 6.3280 */

#define CIMBA_B200_MODEL_AWACS 15    /* tutorial/tut_5_1.c (BASELINE config 5), one trial per warp: 1000 ground targets cycling hiding ->
                                    * staging -> firing -> driving, a radar ticking every second through a five-stage float32 detection
                                    * chain (swept sector, horizon, nadir hole, terrain ray-march, clutter-limited probability with a
                                    * cmb_random_bernoulli draw), the platform on its racetrack, the progress-bar process, the end event
                                    * after num_objects SECONDS.  The terrain map all trials share is registered once per device with
                                    * cimba_b200_awacs_set_terrain(); arr_mean / srv_mean are not used.  Results: objects = targets found
                                    * (struct trial.num_found), sum_wait = sum of the targets' final x, counters[0..5] = targets per
                                    * detect state, [6] = targets per mode (4 x 16 bits), [7] = terrain cells read by the line-of-sight marches; the per-target
                                    * state stays in the workspace (layout: CIMBA_B200_AWACS_* below).  Device-resident interface only.
                                    * Parity with the reference (glibc libm): atan2f / sinf / cosf are restated exactly, powf / expf rounded
                                    * once from double - exact until one of those straddles a test threshold, statistical beyond (DESIGN.md 3.6) */

#define CIMBA_B200_MODEL_RENEGE 16   /* cimba_b200/models/renege_model.cuh, written against the device authoring surface
                                    * (cimba_b200/csrc/cmb_device.cuh) and run by the general engine: `servers` impatient customer
                                    * PROCESSES (a thousand and more) with priorities 0..3 think (mean arr_mean), then ask a
                                    * cmb_resourcepool of (servers + 7) / 8 clerks for a unit with a patience timer running
                                    * (cmb_process_timer_add, mean params[0], default srv_mean): served in time -> timers_clear,
                                    * service (mean srv_mean), release; else the timer resumes the waiter and the acquire unwinds.
                                    * End event at t = num_objects stops everybody.  counters: [0] served [1] reneged [2] other
                                    * signals [3] clerks busy at the end [4] stale wait-list entries [5] log2 of the event list's
                                    * final capacity [6] its key map active [7] processes.  sum_wait = time in line of the served */

#define CIMBA_B200_MODEL_POOL_RECORDED 18 /* cimba_b200/models/cheese_model.cuh = test/test_resourcepool.c as it stands, on the general
                                    * engine: three mice (cmb_process_priority_set + acquire 1..10 units), two rats (pre-empt), a cat
                                    * interrupting them (cmb_random_flip), a pool of `servers` units with its usage history on, end
                                    * event at t = num_objects.  counters[0..7] = the history's cmb_wtdsummary {count, min, max, m1,
                                    * m2, m3, m4, wsum} (count as u64, the rest as bit patterns); objects = successful acquisitions.
                                    * 20 units, 100 time units and the golden seed give test/reference/resourcepool.txt's
                                    * "N 120  Mean 19.77  StdDev 1.147  Variance 1.316  Skewness -6.626  Kurtosis 46.75" */
#define CIMBA_B200_MODEL_TUTORIAL1 19    /* cimba_b200/models/tutorial1_model.cuh = the trial of tutorial/tut_1_7.c (run_MM1_trial :155-222): M/M/1 in a
                                          * cmb_buffer, level history on from params[0] (warm-up time) for num_objects time units, end event of
                                          * priority -100; arr_mean / srv_mean = 1 / arr_rate, 1 / srv_rate; counters[0..7] = the history's
                                          * cmb_wtdsummary (counters[3] = the tutorial's avg_queue_length, as a double's bits).  Runs on the static tier
                                          * (cmb_static.cuh: two processes, a buffer, three events of its own); CIMBA_B200_VARIANT_GENERAL = general engine. */
#define CIMBA_B200_MODEL_PARK 20         /* cimba_b200/models/park_model.cuh = the reference's third tutorial, tutorial/tut_3_1.c: a theme park of nine
                                          * attractions (11 cmb_priorityqueues, 14 batch servers), visitors as processes that balk, jockey and
                                          * renege on patience timers, gold-card priorities, Vose alias routing, PERT rides; 16 simulated hours.
                                          * No parameters (the park is the tutorial's hard-coded one).  counters[0..4] = the tutorial's five
                                          * results - mean time in park, riding, waiting, walking, mean number of rides - as doubles' bits,
                                          * [5] = visitors departed; objects = visitors created.  General engine. */
#define CIMBA_B200_MODEL_TUTORIAL2 21    /* cimba_b200/models/tutorial2_model.cuh = the reference's second tutorial, tutorial/tut_2_1.c: five mice
                                          * acquiring, two rats pre-empting, a cat interrupting, 20 units of cheese, 100 000 time units.  No
                                          * parameters.  counters[0] = the random stream's next raw output after the run, [1] = units in use at
                                          * the end, [2] = objects = successful acquires + pre-empts.  General engine. */

/* Models of your own: write them against cimba_b200/csrc/cmb_device.cuh, end the .cu file with
 * CMB_EXPORT_MODEL(YourModel, "name"), build it with scripts/build_model.py (nvcc, sm_90a) and load the library: */
#define CIMBA_B200_MODEL_USER_BASE 1000
/* Returns a model id >= CIMBA_B200_MODEL_USER_BASE usable wherever a CIMBA_B200_MODEL_* is (device jobs and
 * cimba_b200_run_experiment alike), or a negative CIMBA_B200_E* code.  The library stays loaded for the process' life. */
int cimba_b200_model_load(const char *path_to_model_library);
/* The name the model registered, or NULL for an id nobody loaded. */
const char *cimba_b200_model_name(int model_id);

/* variant 16 of MODEL_MM1 / MODEL_GG1 / MODEL_MMC / MODEL_HOLD / MODEL_HARBOR: the same model as
 * cimba_b200/models/{mm1,gg1,mmc,hold_general,harbor_general}_model.cuh
 * run by the general engine (growable event list, wait lists and queues; any number of servers).  The fast kernels' repair pass
 * and MODEL_MMC with more than 14 servers use it too. */
#define CIMBA_B200_VARIANT_GENERAL 16
/* CIMBA_B200_MODEL_MM1 / _GG1 / _MM1_RECORDED from their authoring-surface source on the static tier (cimba_b200/csrc/cmb_static.cuh):
 * process records and event slots in registers, the queue in shared memory; what it flags is re-run on the general engine.
 * Also CIMBA_B200_MODEL_RESOURCE_RECORDED, _POOL_RECORDED and _TUTORIAL2 on the tier's form with priorities, interrupts and
 * pre-emption (same workspace as their default route; the default routes are unchanged), and CIMBA_B200_MODEL_GUARDED,
 * _GUARDED_RECORDED, _PRIOQ_RECORDED and _PRIOQ with the tier's priority queue and condition (the same workspace as their default
 * route at every capacity; a queue beyond the tier's tables is re-run on the general engine), and CIMBA_B200_MODEL_TIMERS with the
 * tier's timers, resume / yield, waits on processes and events and observers (same workspace as its default route; a trial that
 * needs a ninth spare event slot, or cancels a waited-on event in an order the tier does not keep, is re-run on the general engine),
 * and CIMBA_B200_MODEL_PREEMPT, _BUFFER and _BUFFER_RECORDED on the tier's form with priorities, interrupts and pre-emption, the
 * buffer's waiters in literal heaps (same workspace as their default route; a trial that needs a fifth spare event slot for model 4,
 * a third for models 5 and 12, is re-run on the general engine) */
#define CIMBA_B200_VARIANT_STATIC 17

/* Error codes */
#define CIMBA_B200_OK         0
#define CIMBA_B200_EINVAL    -1  /* bad argument */
#define CIMBA_B200_ENODEVICE -2  /* no usable CUDA device */
#define CIMBA_B200_ECUDA     -3  /* CUDA runtime error; see cimba_b200_last_error() */
#define CIMBA_B200_ETRIAL    -4  /* at least one trial reported a non-zero status */
#define CIMBA_B200_ENOMEM    -5

/* Per-trial status bits (0 = ok).  Bits 1, 2, 8 and 16 are what a fixed-capacity kernel (the fused M/M/1, G/G/1, M/M/c kernels,
 * the static tier, the round-1 coverage kernels) sets when a trial outgrows its tables: the launch re-runs such trials on the
 * general engine by itself, so a caller only sees them with status == NULL (no repair possible) or variant 1.  Bit 4: the fused
 * kernels keep event keys in 30 bits (the reference: 64) - a trial of more than 2^30 events is flagged, not repaired (the general
 * engine has 64-bit keys but would need hours for such a trial).  Bit 64: the general engine's growth arena ran out -
 * pass a larger workspace (cimba_b200_workspace_bytes sizes it for the model's declared need). */
#define CIMBA_B200_TRIAL_QUEUE_OVERFLOW 1u
#define CIMBA_B200_TRIAL_FEL_OVERFLOW   2u
#define CIMBA_B200_TRIAL_KEY_OVERFLOW   4u
#define CIMBA_B200_TRIAL_GUARD_OVERFLOW 8u
#define CIMBA_B200_TRIAL_PROC_OVERFLOW  16u
#define CIMBA_B200_TRIAL_NEGATIVE_HOLD  32u
#define CIMBA_B200_TRIAL_ARENA_EXHAUSTED 64u   /* general engine: a container could not grow (workspace too small) */
#define CIMBA_B200_TRIAL_BAD_ARGUMENT   128u   /* model code: cmb_random_loaded_dice / _hyperexponential with n = 0, or
                                                  cmb_random_alias_create with n = 0 or n above the table's capacity */

/* How trials map onto the machine.  LANE: one trial per CUDA thread (32 trials
 * advance per warp instruction; the default for models whose per-trial state is
 * a few dozen bytes).  WARP: one trial per warp with lane 0 as the dispatcher
 * (the mapping BASELINE.json's north_star names; kept for models with large
 * event lists and for the measured comparison in DESIGN.md). */
#define CIMBA_B200_MAP_LANE 1
#define CIMBA_B200_MAP_WARP 32

/* ------------------------------------------------------------------------
 * Device-resident interface: all pointers are DEVICE pointers; the launch is
 * asynchronous on `stream` (a cudaStream_t passed as void*, NULL = default
 * stream).  This is the hot path proper.
 * ---------------------------------------------------------------------- */
typedef struct cimba_b200_device_job {
    int32_t  model;             /* CIMBA_B200_MODEL_* */
    int32_t  servers;           /* pool capacity for MODEL_MMC, ignored otherwise */
    int32_t  mapping;           /* CIMBA_B200_MAP_LANE (default if 0) or _WARP */
    int32_t  variant;           /* 0 = default kernel; 1 = the unfused formulation (queue_model.cuh), kept for A/B measurement */
    uint64_t master_seed;
    uint64_t first_trial;       /* global index of trial 0 of this job (sharding) */
    uint64_t num_trials;
    uint64_t num_objects;       /* customers generated per trial (NUM_OBJECTS, benchmark/MM1_multi.c:26) */
    /* per-trial parameters, [num_trials] doubles each (struct trial.arr_mean / .srv_mean) */
    const double *arr_mean;
    const double *srv_mean;
    /* per-trial results, [num_trials] each; any may be NULL */
    uint64_t *events;           /* future-event-list pops = cmb_event_execute_next() calls */
    uint64_t *objects;          /* struct trial.obj_cnt */
    double   *t_end;            /* cmb_time() when the event list ran dry */
    double   *sum_wait;         /* struct trial.sum_wait */
    uint32_t *status;           /* CIMBA_B200_TRIAL_* bits */
    uint32_t *max_queue;        /* diagnostic: longest queue seen (MODEL_MMC: most customers alive; MODEL_GUARDED: deepest event list) */
    uint64_t *counters;         /* [num_trials][8] model counters (MODEL_GUARDED: puts, gets, interrupted holds/puts/gets,
                                 * sum of signals, final queue length, interrupts issued); may be NULL */
    /* scratch in HBM for queue/wait-list spill; size from cimba_b200_workspace_bytes() */
    void     *workspace;
    uint64_t  workspace_bytes;
    /* optional pop trace: the first trace_cap pops of EVERY trial, row-major
     * [num_trials][trace_cap]; NULL / 0 to disable */
    uint64_t  trace_cap;
    uint64_t *trace_key;        /* cmb_event_current() after each pop */
    double   *trace_time;       /* cmb_time() after each pop */
    /* capacity of the per-trial HBM ring behind the 32-entry on-chip window of the cmb_objectqueue (M/M/1, G/G/1)
     * and of the resource pool's wait list (M/M/c): a power of two, 0 = the default (512).  The reference's queue
     * is CMB_UNLIMITED (benchmark/MM1_multi.c:103): a trial that outgrows window + ring is not lost - it is re-run
     * on the growable general engine by a repair pass inside the same launch (see DESIGN.md) - but a ring sized for
     * the traffic (rho -> 1) keeps such trials on the fast kernel.  cimba_b200_workspace_bytes() honours it. */
    uint32_t  queue_spill_cap;
    uint32_t  reserved0;        /* 0 */
    /* optional DEVICE pointer to 4 uint64 the simulation kernel ADDS to (zero them first): [0] event-loop
     * iterations summed over warps, [1] warps that ran, [2] trials the repair pass re-ran, [3] reserved.
     * bench.py turns [0] into issued warp-instructions with the loop's calibrated instruction count. */
    uint64_t *diag;
    /* experiment-wide model parameters for models built with the device authoring API (include/cmb_device.cuh):
     * HOST pointer to num_params <= CIMBA_B200_MAX_MODEL_PARAMS doubles, copied at launch; NULL / 0 otherwise */
    const double *params;
    uint32_t  num_params;
    uint32_t  reserved1;        /* 0 */
} cimba_b200_device_job;
#define CIMBA_B200_MAX_MODEL_PARAMS 16

/* MODEL_AWACS: the terrain every trial reads (struct terrain, tutorial/tut_5_1.c:96-108, as terrain_init :197-294 fills
 * it).  map is a DEVICE pointer to rows x cols float32 elevations, row-major, and must stay valid while jobs run.
 * Registered per CUDA device (the current one); later launches of MODEL_AWACS on that device use it. */
typedef struct cimba_b200_awacs_terrain {
    const float *map;
    uint32_t cols, rows;
    float x_scale, y_scale;         /* metres per arc-second */
    float x_min, x_max, y_min, y_max;
} cimba_b200_awacs_terrain;
int cimba_b200_awacs_set_terrain(const cimba_b200_awacs_terrain *terrain);
/* The same for a caller without CUDA code of its own: `terrain->map` is a HOST pointer (tp->map as terrain_init left
 * it); the library keeps a device copy per GPU (replaced by the next upload, freed by cimba_b200_release_cache). */
int cimba_b200_awacs_upload_terrain(const cimba_b200_awacs_terrain *terrain);

/* MODEL_AWACS workspace: per trial CIMBA_B200_AWACS_STATE_BYTES, columns of CIMBA_B200_AWACS_STRIDE entries in this
 * order: float x, y, alt, dir, vel, time_s, rcs_now; uint32 flags (bits 0-1 mode, 4-6 detect state, 8 found);
 * uint32 wake_key; double wake_t.  Entries 0..999 are the targets. */
#define CIMBA_B200_AWACS_TARGETS 1000
#define CIMBA_B200_AWACS_STRIDE 1024
#define CIMBA_B200_AWACS_STATE_BYTES (CIMBA_B200_AWACS_STRIDE * (7 * 4 + 4 + 4 + 8))

/* Bytes of HBM scratch the job needs (0 is possible). */
uint64_t cimba_b200_workspace_bytes(const cimba_b200_device_job *job);

/* Enqueue the persistent simulation kernel for the job.  Asynchronous. */
int cimba_b200_launch(const cimba_b200_device_job *job, void *stream);

/* Number of kernels this library has launched so far in this process. */
uint64_t cimba_b200_launch_count(void);

/* CTAs of the M/M/1 trial kernel (MODEL_MM1, variant 0; trace != 0: its pop-recording form) resident per SM of the
 * current device, with the shared-memory carveout the library asks for before it launches them: a diagnostic.
 * Negative: an error code. */
int cimba_b200_mm1_resident_ctas(int trace);

/* Reduce per-trial results to a cmb_datasummary of avg = sum_wait/objects on
 * the device (benchmark/MM1_multi.c:143-148 does this with a serial host loop).
 * out_summary: DEVICE pointer to 8 doubles {count, min, max, m1, m2, m3, m4, 0}.
 * Deterministic (fixed merge tree, cmb_datasummary_merge arithmetic). */
int cimba_b200_summarize(const double *sum_wait, const uint64_t *objects,
                         uint64_t num_trials, double *out_summary, void *stream);

/* cmb_wtdsummary_add (src/cmb_wtdsummary.c:82-137) over n device-resident (x, w) pairs.
 * out_row: DEVICE pointer to 8 words {count (u64), min, max, m1, m2, m3, m4, wsum (f64 bit
 * patterns)} - the row format MODEL_MM1_RECORDED writes per trial. */
int cimba_b200_summarize_weighted(const double *x, const double *w, uint64_t n,
                                  uint64_t *out_row, void *stream);

/* cmb_wtdsummary_merge (src/cmb_wtdsummary.c:152-194) over n device-resident rows of that
 * format (one per trial) into one row: the per-GPU step before the NCCL all-gather. */
int cimba_b200_merge_weighted_rows(const uint64_t *rows, uint64_t n, uint64_t *out_row, void *stream);
/* All three reductions refuse an empty input: num_trials / n = 0 returns CIMBA_B200_EINVAL, launches nothing and leaves
 * the output untouched (an empty summary is what *_initialize gives on the host). */

/* ------------------------------------------------------------------------
 * Host-buffer interface = the cimba_run_experiment() replacement.
 * ---------------------------------------------------------------------- */
#define CIMBA_B200_NO_FIELD ((size_t)-1)

typedef struct cimba_b200_experiment {
    int32_t  model;
    int32_t  servers;
    int32_t  mapping;           /* 0 = default */
    int32_t  device;            /* CUDA device ordinal, -1 = current */
    int32_t  variant;           /* kernel variant, as cimba_b200_device_job.variant (0 = default) */
    uint32_t queue_spill_cap;   /* as cimba_b200_device_job.queue_spill_cap (0 = default) */
    uint64_t master_seed;
    uint64_t first_trial;
    uint64_t num_objects;
    /* byte offsets of the fields inside one trial struct */
    size_t off_arr_mean;        /* double, in  (required) */
    size_t off_srv_mean;        /* double, in  (required) */
    size_t off_obj_cnt;         /* uint64, out (or NO_FIELD) */
    size_t off_sum_wait;        /* double, out (or NO_FIELD) */
    size_t off_avg_wait;        /* double, out = sum_wait / obj_cnt (or NO_FIELD) */
    size_t off_events;          /* uint64, out (or NO_FIELD) */
    size_t off_t_end;           /* double, out (or NO_FIELD) */
    size_t off_status;          /* uint32, out (or NO_FIELD) */
    size_t off_max_queue;       /* uint32, out (or NO_FIELD): longest queue / deepest list / most ships alive */
    size_t off_counters;        /* uint64[8], out (or NO_FIELD): the model's counters (see CIMBA_B200_MODEL_*) */
    /* the model's scalar parameters, as cimba_b200_device_job.params: HOST pointer to num_params doubles (or NULL, 0) -
     * e.g. the warm-up time of CIMBA_B200_MODEL_TUTORIAL1, the patience of CIMBA_B200_MODEL_RENEGE */
    const double *params;
    uint32_t num_params;
    uint32_t reserved;
} cimba_b200_experiment;

/* Blocks until all trials are done; results written into the caller's array.
 * Returns CIMBA_B200_ETRIAL if any trial's status is non-zero (results of the
 * other trials are still valid). */
int cimba_b200_run_experiment(void *your_experiment_array,
                              uint64_t num_trials,
                              size_t trial_struct_size,
                              const cimba_b200_experiment *desc);

/* cimba_b200_run_experiment keeps its pinned staging buffers, device arena and stream per device
 * between calls (grow-only).  This frees them (the analogue of the reference's per-thread mempools
 * being torn down at thread exit, src/cimba.c:134-139). */
void cimba_b200_release_cache(void);

/* The same, sharded over every visible GPU (or the first max_gpus > 0 of them): one host
 * thread per GPU runs a contiguous block of the array - the counterpart of the
 * reference executive's one pthread per core (src/cimba.c:171-182).  Results do not
 * depend on the GPU count (seeds are a function of the global trial index). */
int cimba_b200_run_experiment_all_gpus(void *your_experiment_array,
                                       uint64_t num_trials,
                                       size_t trial_struct_size,
                                       const cimba_b200_experiment *desc,
                                       int max_gpus);

/* cimba_set_thread_hooks / cimba_thread_context (include/cimba.h:148-195, src/cimba.c:65-78, :97-140; CHANGELOG: "for
 * managing CUDA streams").  The reference calls init(usrarg, tid) at the start of each of its worker pthreads, keeps
 * the returned pointer as that thread's context and calls exit(context) before the thread ends.  Here the worker
 * threads are the ones cimba_b200_run_experiment_all_gpus starts, one per GPU, and tid is the GPU's ordinal: the
 * hooks run on that thread after cudaSetDevice(tid) and before / after its block of trials.
 * cimba_b200_run_experiment runs on the caller's own thread and calls no hook. */
typedef void *(cimba_b200_thread_init_func)(void *usrarg, uint64_t tid);
typedef void (cimba_b200_thread_exit_func)(void *thrctx);
void  cimba_b200_set_thread_hooks(cimba_b200_thread_init_func *initfunc, void *usrarg,
                                  cimba_b200_thread_exit_func *exitfunc);
void *cimba_b200_thread_context(void);

/* ------------------------------------------------------------------------
 * cmb_datasummary on the host (reference include/cmb_datasummary.h:42-51,
 * src/cmb_datasummary.c:93-166): same field order and arithmetic, used to fold
 * per-GPU summaries after the NCCL all-gather.
 * ---------------------------------------------------------------------- */
typedef struct cimba_b200_datasummary {
    uint64_t cookie;
    uint64_t count;
    double   min, max;
    double   m1, m2, m3, m4;
} cimba_b200_datasummary;

void     cimba_b200_datasummary_initialize(cimba_b200_datasummary *dsp);
uint64_t cimba_b200_datasummary_add(cimba_b200_datasummary *dsp, double y);
uint64_t cimba_b200_datasummary_merge(cimba_b200_datasummary *tgt,
                                      const cimba_b200_datasummary *dsp1,
                                      const cimba_b200_datasummary *dsp2);
double   cimba_b200_datasummary_mean(const cimba_b200_datasummary *dsp);
double   cimba_b200_datasummary_variance(const cimba_b200_datasummary *dsp);
double   cimba_b200_datasummary_stddev(const cimba_b200_datasummary *dsp);
/* include/cmb_datasummary.h:133-179 (count / max / min), src/cmb_datasummary.c:214-249 (sample skewness and
 * sample excess kurtosis with the finite-sample corrections), :168-212 (print: "N", "Mean", "StdDev", "Variance",
 * "Skewness", "Kurtosis" as %#8.4g, each only when the count supports it; lead_ins = 0 prints tab-separated). */
uint64_t cimba_b200_datasummary_count(const cimba_b200_datasummary *dsp);
double   cimba_b200_datasummary_max(const cimba_b200_datasummary *dsp);
double   cimba_b200_datasummary_min(const cimba_b200_datasummary *dsp);
double   cimba_b200_datasummary_skewness(const cimba_b200_datasummary *dsp);
double   cimba_b200_datasummary_kurtosis(const cimba_b200_datasummary *dsp);
void     cimba_b200_datasummary_print(const cimba_b200_datasummary *dsp, FILE *fp, int lead_ins);

/* cmb_wtdsummary (include/cmb_wtdsummary.h:41-44: the data summary plus the sum of weights;
 * src/cmb_wtdsummary.c:82-137 add, :152-194 merge).  Same arithmetic as the device kernels. */
typedef struct cimba_b200_wtdsummary {
    cimba_b200_datasummary base;
    double   wsum;
} cimba_b200_wtdsummary;

void     cimba_b200_wtdsummary_initialize(cimba_b200_wtdsummary *wsp);
uint64_t cimba_b200_wtdsummary_add(cimba_b200_wtdsummary *wsp, double x, double w);
uint64_t cimba_b200_wtdsummary_merge(cimba_b200_wtdsummary *tgt,
                                     const cimba_b200_wtdsummary *ws1,
                                     const cimba_b200_wtdsummary *ws2);
double   cimba_b200_wtdsummary_mean(const cimba_b200_wtdsummary *wsp);
double   cimba_b200_wtdsummary_variance(const cimba_b200_wtdsummary *wsp);
/* include/cmb_wtdsummary.h:208-250 and src/cmb_wtdsummary.c (print): all delegate to the data summary part. */
double   cimba_b200_wtdsummary_stddev(const cimba_b200_wtdsummary *wsp);
double   cimba_b200_wtdsummary_skewness(const cimba_b200_wtdsummary *wsp);
double   cimba_b200_wtdsummary_kurtosis(const cimba_b200_wtdsummary *wsp);
void     cimba_b200_wtdsummary_print(const cimba_b200_wtdsummary *wsp, FILE *fp, int lead_ins);

/* cmb_random_fmix64 (src/cmb_random.c:70-80): per-trial seed derivation. */
uint64_t cimba_b200_fmix64(uint64_t seed, uint64_t nonce);

/* Device-side variate generation for stream KATs: n draws from the stream
 * seeded with `seed`, written to the DEVICE buffer `out` (n doubles).
 * kind: 0 raw sfc64 bits, 1 exponential(p0), 2 std_normal, 3 uniform01,
 *       4 normal(p0,p1), 5 erlang((unsigned)p0, p1), 6 uniform(p0,p1),
 *       7 dice((long)p0,(long)p1), 8 bernoulli(p0) */
int cimba_b200_rng_draws(uint64_t seed, int kind, double p0, double p1,
                         uint64_t n, double *out, void *stream);

/* The rest of cmb_random (include/cmb_random.h:189-940) on the device, same calling form:
 * kind  9 triangular(min,mode,max)   10 lognormal(m,s)        11 logistic(m,s)     12 cauchy(mode,scale)
 *      13 hypoexponential(n, m[n])   14 hyperexponential(n, m[n], p[n])            15 gamma(shape,scale)
 *      16 beta(a,b,min,max)          17 PERT(min,mode,max)    18 weibull(shape,scale)  19 pareto(shape,mode)
 *      20 chisquared(k)              21 F_dist(a,b)           22 t_dist(m,s,v)     23 rayleigh(s)
 *      24 flip()                     25 geometric(p)          26 binomial(n,p)     27 negative_binomial(m,p)
 *      28 poisson(r)                 29 loaded_dice(n, p[n])  30 alias_sample over alias_create(n, p[n])
 *      31 std_gamma(shape)           32 PERT_mod(min,mode,max,lambda)              33 pascal(m,p)
 * params: HOST array of num_params <= CIMBA_B200_RNG_MAX_PARAMS doubles; out: DEVICE buffer of n doubles. */
#define CIMBA_B200_RNG_MAX_PARAMS 16
int cimba_b200_rng_draws_ex(uint64_t seed, int kind, const double *params, uint32_t num_params,
                            uint64_t n, double *out, void *stream);

/* cmb_random_alias_create (src/cmb_random.c:688-752): Vose alias tables for n alternatives with
 * probabilities pa[n], written to the caller's uprob[n] / alias[n] (host memory; upload them for
 * device-side alias sampling). */
int cimba_b200_alias_create(uint32_t n, const double *pa, uint64_t *uprob, uint32_t *alias);

const char *cimba_b200_version(void);
const char *cimba_b200_last_error(void);
int         cimba_b200_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* CIMBA_B200_H */
