/*
 * repair_driver.c - TEST INFRASTRUCTURE ONLY.
 *
 * The machine shop of examples/repair_model.cuh written against the UNMODIFIED reference library (compiled by
 * oracle/Makefile into oracle/_ref/libcimba_ref.so; this file is built into oracle/_ref/librepairdrv.so by
 * oracle/repair.mk).  It is the oracle of the shop on both engines: tests/golden/make_repair_golden.py makes the stored
 * vectors from it, and tests/test_static_resources.py / tests/test_gpu_static_resources.py compare with it live.
 *
 * `machines` machines share a crew of `servers` units (its usage history on) and one bench.  Machine i, num_objects
 * times: up time (exponential, arr_mean); acquire need = 1 + (i & 1) crew (1 with a crew of one); repair (exponential,
 * srv_mean); release; the bench for an inspection (exponential, srv_mean / 4).  With exit_holding the last cycle ends
 * with cmb_process_exit right after the repair, the crew still held.
 * objects = repairs, sum_wait = total downtime, counter[0] = acquisitions that found 0 < available < need, counter[1] =
 * bench acquisitions that found it held, counter[2..6] = the crew history's count, m1, m2, wsum, max (bit patterns).
 * Seeds and event counting as oracle/ref_build/ref_driver.c: trial i is seeded cmb_random_fmix64(master, i), an event is
 * one successful cmb_event_execute_next().
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <cimba.h>

struct repair_result {          /* the layout of ref_driver.c's struct ref_result (tests/oracle_libs.py: Result) */
    uint64_t events;
    uint64_t objects;
    double t_end;
    double sum_wait;
    uint64_t max_fel;
    uint64_t max_queue;
    uint64_t counter[8];
};

struct rp_world;

struct rp_machine {
    struct rp_world *world;
    unsigned index;
};

struct rp_world {
    int servers;
    uint64_t num_objects;
    double arr_mean, srv_mean;
    int exit_holding;
    struct cmb_resourcepool *crew;
    struct cmb_resource *bench;
    struct repair_result *res;
};

static void *rp_machine_body(struct cmb_process *me, void *vm)
{
    cmb_unused(me);
    struct rp_machine *mc = vm;
    struct rp_world *w = mc->world;
    const uint64_t need = w->servers >= 2 ? 1u + (mc->index & 1u) : 1u;
    for (uint64_t k = 0u; k < w->num_objects; k++) {
        (void)cmb_process_hold(cmb_random_exponential(w->arr_mean));
        const double failed = cmb_time();
        const uint64_t avail = cmb_resourcepool_available(w->crew);
        if (avail > 0u && avail < need) {
            w->res->counter[0] += 1u;
        }
        (void)cmb_resourcepool_acquire(w->crew, need);
        (void)cmb_process_hold(cmb_random_exponential(w->srv_mean));
        if (w->exit_holding && k + 1u == w->num_objects) {
            cmb_process_exit(NULL);
        }
        cmb_resourcepool_release(w->crew, need);
        if (cmb_resource_in_use(w->bench) != 0u) {
            w->res->counter[1] += 1u;
        }
        (void)cmb_resource_acquire(w->bench);
        (void)cmb_process_hold(cmb_random_exponential(0.25 * w->srv_mean));
        cmb_resource_release(w->bench);
        w->res->sum_wait += cmb_time() - failed;
        w->res->objects += 1u;
    }
    return NULL;
}

static void run_repair_trial(uint64_t seed, int servers, uint64_t num_objects, double arr_mean, double srv_mean,
                             unsigned machines, int exit_holding, uint64_t trace_cap, uint64_t *trace_key,
                             double *trace_time, struct repair_result *res)
{
    memset(res, 0, sizeof(*res));
    cmb_logger_flags_off(CMB_LOGGER_INFO);
    cmb_random_initialize(seed);
    cmb_event_queue_initialize(0.0);

    struct rp_world w = { .servers = servers, .num_objects = num_objects, .arr_mean = arr_mean, .srv_mean = srv_mean,
                          .exit_holding = exit_holding, .res = res };
    w.crew = cmb_resourcepool_create();
    cmb_resourcepool_initialize(w.crew, "Crew", (uint64_t)servers);
    cmb_resourcepool_start_recording(w.crew);
    w.bench = cmb_resource_create();
    cmb_resource_initialize(w.bench, "Bench");
    struct rp_machine *mach = calloc(machines, sizeof(*mach));
    struct cmb_process **proc = calloc(machines, sizeof(*proc));
    for (unsigned i = 0u; i < machines; i++) {
        mach[i].world = &w;
        mach[i].index = i;
        proc[i] = cmb_process_create();
        cmb_process_initialize(proc[i], "Machine", rp_machine_body, &mach[i], 0);
        cmb_process_start(proc[i]);
    }

    uint64_t n = 0u;
    while (cmb_event_execute_next()) {
        if (n < trace_cap) {
            trace_key[n] = cmb_event_current();
            trace_time[n] = cmb_time();
        }
        n++;
    }
    res->events = n;
    res->t_end = cmb_time();

    cmb_resourcepool_stop_recording(w.crew);
    struct cmb_wtdsummary ws;
    cmb_wtdsummary_initialize(&ws);
    (void)cmb_timeseries_summarize(cmb_resourcepool_get_history(w.crew), &ws);
    const struct cmb_datasummary *ds = (const struct cmb_datasummary *)&ws;
    const double v[4] = { ds->m1, ds->m2, ws.wsum, ds->max };
    res->counter[2] = ds->count;
    memcpy(&res->counter[3], v, sizeof(v));
    for (unsigned i = 0u; i < machines; i++) {
        cmb_process_terminate(proc[i]);
        cmb_process_destroy(proc[i]);
    }
    free(proc);
    free(mach);
    cmb_resource_destroy(w.bench);
    cmb_resourcepool_destroy(w.crew);
    cmb_event_queue_terminate();
}

/* trials [first, first + count), seeds cmb_random_fmix64(master_seed, global trial index), serially */
int repair_ref_run_trials(int servers, uint64_t master_seed, uint64_t first, uint64_t count, uint64_t num_objects,
                          double arr_mean, double srv_mean, unsigned machines, int exit_holding, struct repair_result *out)
{
    for (uint64_t i = 0u; i < count; i++) {
        run_repair_trial(cmb_random_fmix64(master_seed, first + i), servers, num_objects, arr_mean, srv_mean, machines,
                         exit_holding, 0u, NULL, NULL, &out[i]);
    }
    return 0;
}

/* one trial of the given seed, with its first trace_cap pops (event handle, time) */
int repair_ref_trace_trial(int servers, uint64_t seed, uint64_t num_objects, double arr_mean, double srv_mean,
                           unsigned machines, int exit_holding, uint64_t trace_cap, uint64_t *trace_key, double *trace_time,
                           struct repair_result *out)
{
    run_repair_trial(seed, servers, num_objects, arr_mean, srv_mean, machines, exit_holding, trace_cap, trace_key, trace_time,
                     out);
    return 0;
}
