/*
 * clinic_driver.c - TEST INFRASTRUCTURE ONLY.
 *
 * The walk-in clinic of examples/clinic_model.cuh written against the UNMODIFIED reference library (compiled by
 * oracle/Makefile into oracle/_ref/libcimba_ref.so; this file is built into oracle/_ref/libclinicdrv.so by oracle/clinic.mk).
 * It is the oracle of the clinic on both engines: tests/golden/make_clinic_golden.py makes the stored vectors from it, and
 * tests/test_model_random.py / tests/test_gpu_clinic.py compare with it live where it was built.
 *
 * num_objects groups arrive, hyperexponential gaps (means arr/2, arr, 2.5 arr; probabilities 0.5, 0.3, 0.2).  A group is
 * geometric(0.6) + binomial(2, 0.25) + negative_binomial(1, 0.8) + pascal(1, 0.9) patients; triage by an alias table
 * (0.5, 0.3, 0.2) sends it to desk 0's queue, to the queue desks 1 and 2 share, or home (counted).  Services: desk 0
 * PERT_mod(srv/4, srv, 3 srv, 4); desk 1 2 srv std_beta(2, 3) + srv/10 chisquared(3) + srv/20 std_gamma(2.5); desk 2
 * srv/2 F(5, 10) + erlang(2, srv/4) + hypoexponential(srv/2, srv)/10.  After each service: a visit code by loaded dice
 * (0.4, 0.3, 0.2, 0.1), cauchy, std_t, t, logistic into one summary, weibull, pareto, gamma(0.5), std_exponential into another.
 * Desk 0's queue length is a weighted summary, sampled before each put to it and before each get from it.
 * objects = patients served, sum_wait = their time in the clinic, max_queue = patients sent home, counter[0..7] = the row of
 * summary `report` (0 queue, 1 signed values, 2 log / pow values, 3 group sizes, 4 visit codes): {count, min, max, m1, m2, m3,
 * m4, wsum} with wsum = count for a data summary.  Every draw is a statement of its own, as in the model.
 * Seeds and event counting as oracle/ref_build/ref_driver.c: trial i is seeded cmb_random_fmix64(master, i), an event is one
 * successful cmb_event_execute_next().
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <cimba.h>

struct clinic_result {          /* the layout of ref_driver.c's struct ref_result (tests/oracle_libs.py: Result) */
    uint64_t events;
    uint64_t objects;
    double t_end;
    double sum_wait;
    uint64_t max_fel;
    uint64_t max_queue;
    uint64_t counter[8];
};

struct cl_world {
    uint64_t num_objects;
    double arr_mean, srv_mean;
    double hyper_m[3], hyper_p[3], hypo_m[2], codes_p[4];
    struct cmb_objectqueue *q0, *q1;
    struct cmb_random_alias *route;
    struct cmb_wtdsummary q0_len;
    struct cmb_datasummary signed_values, logpow_values, sizes, codes;
    double q0_since, sum_wait;
    uint64_t served, advised;
};

struct cl_desk {
    struct cl_world *world;
    unsigned index;
};

static void q0_sample(struct cl_world *w)
{
    (void)cmb_wtdsummary_add(&w->q0_len, (double)cmb_objectqueue_length(w->q0), cmb_time() - w->q0_since);
    w->q0_since = cmb_time();
}

static void *cl_arrival(struct cmb_process *me, void *vw)
{
    cmb_unused(me);
    struct cl_world *w = vw;
    for (uint64_t g = 0u; g < w->num_objects; g++) {
        (void)cmb_process_hold(cmb_random_hyperexponential(3u, w->hyper_m, w->hyper_p));
        uint64_t size = cmb_random_geometric(0.6);
        size += cmb_random_binomial(2u, 0.25);
        size += cmb_random_negative_binomial(1u, 0.8);
        size += cmb_random_pascal(1u, 0.9);
        (void)cmb_datasummary_add(&w->sizes, (double)size);
        const unsigned desk = cmb_random_alias_sample(w->route);
        if (desk == 2u) {
            w->advised += size;
            continue;
        }
        for (uint64_t k = 0u; k < size; k++) {
            const double now = cmb_time();
            uint64_t stamp;
            memcpy(&stamp, &now, sizeof stamp);
            if (desk == 0u) {
                q0_sample(w);
                (void)cmb_objectqueue_put(w->q0, (void *)(uintptr_t)stamp);
            }
            else {
                (void)cmb_objectqueue_put(w->q1, (void *)(uintptr_t)stamp);
            }
        }
    }
    return NULL;
}

static double cl_service(struct cl_world *w, unsigned d)
{
    const double srv = w->srv_mean;
    if (d == 0u) {
        return cmb_random_PERT_mod(0.25 * srv, srv, 3.0 * srv, 4.0);
    }
    if (d == 1u) {
        const double b = cmb_random_std_beta(2.0, 3.0);
        const double c = cmb_random_chisquared(3.0);
        const double g = cmb_random_std_gamma(2.5);
        return 2.0 * srv * b + 0.1 * srv * c + 0.05 * srv * g;
    }
    const double f = cmb_random_F_dist(5.0, 10.0);
    const double e = cmb_random_erlang(2u, 0.25 * srv);
    const double h = cmb_random_hypoexponential(2u, w->hypo_m);
    return 0.5 * srv * f + e + 0.1 * h;
}

static void *cl_desk_body(struct cmb_process *me, void *vd)
{
    cmb_unused(me);
    struct cl_desk *dk = vd;
    struct cl_world *w = dk->world;
    for (;;) {
        void *obj = NULL;
        if (dk->index == 0u) {
            q0_sample(w);
            (void)cmb_objectqueue_get(w->q0, &obj);
        }
        else {
            (void)cmb_objectqueue_get(w->q1, &obj);
        }
        (void)cmb_process_hold(cl_service(w, dk->index));
        const uint64_t stamp = (uint64_t)(uintptr_t)obj;
        double t0;
        memcpy(&t0, &stamp, sizeof t0);
        w->sum_wait += cmb_time() - t0;
        w->served += 1u;
        (void)cmb_datasummary_add(&w->codes, (double)cmb_random_loaded_dice(4u, w->codes_p));
        (void)cmb_datasummary_add(&w->signed_values, cmb_random_cauchy(0.0, 1.0));
        (void)cmb_datasummary_add(&w->signed_values, cmb_random_std_t_dist(4.0));
        (void)cmb_datasummary_add(&w->signed_values, cmb_random_t_dist(1.0, 2.0, 5.0));
        (void)cmb_datasummary_add(&w->signed_values, cmb_random_logistic(0.0, 1.0));
        (void)cmb_datasummary_add(&w->logpow_values, cmb_random_weibull(1.5, w->srv_mean));
        (void)cmb_datasummary_add(&w->logpow_values, cmb_random_pareto(3.0, 1.0));
        (void)cmb_datasummary_add(&w->logpow_values, cmb_random_gamma(0.5, 1.0));
        (void)cmb_datasummary_add(&w->logpow_values, cmb_random_std_exponential());
    }
    return NULL;
}

static void put_row(const struct cmb_datasummary *ds, double wsum, uint64_t *row)
{
    const double v[7] = { ds->min, ds->max, ds->m1, ds->m2, ds->m3, ds->m4, wsum };
    row[0] = ds->count;
    memcpy(&row[1], v, sizeof v);
}

static void run_clinic_trial(uint64_t seed, uint64_t num_objects, double arr_mean, double srv_mean, unsigned report,
                             uint64_t trace_cap, uint64_t *trace_key, double *trace_time, struct clinic_result *res)
{
    memset(res, 0, sizeof(*res));
    cmb_logger_flags_off(CMB_LOGGER_INFO);
    cmb_random_initialize(seed);
    cmb_event_queue_initialize(0.0);

    struct cl_world w;
    memset(&w, 0, sizeof w);
    w.num_objects = num_objects;
    w.arr_mean = arr_mean;
    w.srv_mean = srv_mean;
    w.hyper_m[0] = 0.5 * arr_mean;
    w.hyper_m[1] = arr_mean;
    w.hyper_m[2] = 2.5 * arr_mean;
    w.hyper_p[0] = 0.5;
    w.hyper_p[1] = 0.3;
    w.hyper_p[2] = 0.2;
    w.hypo_m[0] = 0.5 * srv_mean;
    w.hypo_m[1] = srv_mean;
    w.codes_p[0] = 0.4;
    w.codes_p[1] = 0.3;
    w.codes_p[2] = 0.2;
    w.codes_p[3] = 0.1;
    const double desks_p[3] = { 0.5, 0.3, 0.2 };
    w.route = cmb_random_alias_create(3u, desks_p);
    cmb_wtdsummary_initialize(&w.q0_len);
    cmb_datasummary_initialize(&w.signed_values);
    cmb_datasummary_initialize(&w.logpow_values);
    cmb_datasummary_initialize(&w.sizes);
    cmb_datasummary_initialize(&w.codes);
    w.q0 = cmb_objectqueue_create();
    cmb_objectqueue_initialize(w.q0, "Desk 0", CMB_UNLIMITED);
    w.q1 = cmb_objectqueue_create();
    cmb_objectqueue_initialize(w.q1, "Desks 1-2", CMB_UNLIMITED);

    struct cmb_process *proc[4];
    struct cl_desk desk[3];
    proc[0] = cmb_process_create();
    cmb_process_initialize(proc[0], "Arrivals", cl_arrival, &w, 0);
    cmb_process_start(proc[0]);
    for (unsigned d = 0u; d < 3u; d++) {
        desk[d].world = &w;
        desk[d].index = d;
        proc[d + 1u] = cmb_process_create();
        cmb_process_initialize(proc[d + 1u], "Desk", cl_desk_body, &desk[d], 0);
        cmb_process_start(proc[d + 1u]);
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
    q0_sample(&w);
    res->objects = w.served;
    res->sum_wait = w.sum_wait;
    res->max_queue = w.advised;
    switch (report) {
    case 1u: put_row(&w.signed_values, (double)w.signed_values.count, res->counter); break;
    case 2u: put_row(&w.logpow_values, (double)w.logpow_values.count, res->counter); break;
    case 3u: put_row(&w.sizes, (double)w.sizes.count, res->counter); break;
    case 4u: put_row(&w.codes, (double)w.codes.count, res->counter); break;
    default: put_row((const struct cmb_datasummary *)&w.q0_len, w.q0_len.wsum, res->counter); break;
    }

    for (unsigned i = 0u; i < 4u; i++) {
        cmb_process_terminate(proc[i]);
        cmb_process_destroy(proc[i]);
    }
    cmb_objectqueue_destroy(w.q1);
    cmb_objectqueue_destroy(w.q0);
    cmb_random_alias_destroy(w.route);
    cmb_event_queue_terminate();
}

/* trials [first, first + count), seeds cmb_random_fmix64(master_seed, global trial index), serially */
int clinic_ref_run_trials(uint64_t master_seed, uint64_t first, uint64_t count, uint64_t num_objects, double arr_mean,
                          double srv_mean, unsigned report, struct clinic_result *out)
{
    for (uint64_t i = 0u; i < count; i++) {
        run_clinic_trial(cmb_random_fmix64(master_seed, first + i), num_objects, arr_mean, srv_mean, report, 0u, NULL, NULL,
                         &out[i]);
    }
    return 0;
}

/* one trial of the given seed, with its first trace_cap pops (event handle, time) */
int clinic_ref_trace_trial(uint64_t seed, uint64_t num_objects, double arr_mean, double srv_mean, unsigned report,
                           uint64_t trace_cap, uint64_t *trace_key, double *trace_time, struct clinic_result *out)
{
    run_clinic_trial(seed, num_objects, arr_mean, srv_mean, report, trace_cap, trace_key, trace_time, out);
    return 0;
}
