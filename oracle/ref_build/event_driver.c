/*
 * event_driver.c - TEST INFRASTRUCTURE ONLY.
 *
 * The sequence of the reference's own event-queue test (test/test_event.c, test_events()) written against the UNMODIFIED
 * reference library (compiled by oracle/Makefile into oracle/_ref/libcimba_ref.so; this file is built into
 * oracle/_ref/libeventdrv.so by oracle/event.mk), without its printing, returning what examples/event_model.cuh's EventTestT
 * reports: tests/golden/make_event_golden.py makes tests/golden/event_vectors.json from it.
 *
 * The queue starts at time 3; nine test_action events (subjects and objects foo, bar, yuk) and end_sim at 100; the event
 * (test_action, bar, foo) is found and cancelled; every test_action of subject yuk is found and cancelled; three more at t = 20,
 * p = 20; (yuk, foo) rescheduled to now + 25, (yuk, bar) reprioritized to 3; the events of subject bar counted, then cancelled;
 * the queue executed until end_sim clears it.  Every test_action reschedules itself at now + exponential(10), priority
 * dice(1, 5).  The row (struct ref_result's layout, tests/oracle_libs.py: Result):
 *   counter[0] the first pattern_find handle   [1] the bits of its cmb_event_time   [2] its cmb_event_priority
 *   counter[3] the handles the wildcard loop cancelled, 16 bits each, the first in the low bits
 *   counter[4] the pattern_count result   [5] the pattern_cancel result   [6] cmb_event_queue_count() before the run
 *   counter[7] test_action events executed
 *   events = events executed, t_end = the clock at the end; objects, sum_wait, max_fel, max_queue = 0.
 * Trial i is seeded cmb_random_fmix64(master, i) as in oracle/ref_build/ref_driver.c.  The pop trace holds each executed
 * event's handle and time, taken as its action starts (cmb_event_current() is 0 once end_sim has cleared the queue).
 */
#include <stdint.h>
#include <string.h>

#include <cimba.h>

struct event_result {
    uint64_t events;
    uint64_t objects;
    double t_end;
    double sum_wait;
    uint64_t max_fel;
    uint64_t max_queue;
    uint64_t counter[8];
};

static const char *evstrs[] = {"foo", "bar", "yuk"};

static uint64_t g_pops, g_actions, g_cap;
static uint64_t *g_keys;
static double *g_times;

static void note_pop(void)
{
    if (g_pops < g_cap) {
        g_keys[g_pops] = cmb_event_current();
        g_times[g_pops] = cmb_time();
    }
    g_pops++;
}

static void test_action(void *subject, void *object)
{
    note_pop();
    g_actions++;
    (void)cmb_event_schedule(test_action, subject, object, cmb_time() + cmb_random_exponential(10),
                             (int16_t)cmb_random_dice(1, 5));
}

static void end_sim(void *subject, void *object)
{
    (void)subject;
    (void)object;
    note_pop();
    cmb_event_queue_clear();
}

static void run_event_trial(uint64_t seed, uint64_t cap, uint64_t *keys, double *times, struct event_result *r)
{
    memset(r, 0, sizeof *r);
    g_pops = g_actions = 0u;
    g_cap = cap;
    g_keys = keys;
    g_times = times;
    cmb_random_initialize(seed);
    cmb_event_queue_initialize(3.0);

    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) {
            const double t = cmb_time() + cmb_random_exponential(10.0);
            const int64_t p = cmb_random_dice(1, 5);
            (void)cmb_event_schedule(test_action, (void *)evstrs[i], (void *)evstrs[j], t, p);
        }
    }
    (void)cmb_event_schedule(end_sim, NULL, NULL, 100.0, 0);

    uint64_t handle = cmb_event_pattern_find(test_action, (void *)evstrs[1], (void *)evstrs[0]);
    const double ht = cmb_event_time(handle);
    r->counter[0] = handle;
    memcpy(&r->counter[1], &ht, sizeof ht);
    r->counter[2] = (uint64_t)cmb_event_priority(handle);
    (void)cmb_event_cancel(handle);

    unsigned n = 0u;
    while ((handle = cmb_event_pattern_find(test_action, (void *)evstrs[2], CMB_ANY_OBJECT))) {
        if (n < 4u) r->counter[3] |= (handle & 0xffffu) << (16u * n);
        n++;
        (void)cmb_event_cancel(handle);
    }

    for (int j = 0; j < 3; j++) {
        (void)cmb_event_schedule(test_action, (void *)evstrs[2], (void *)evstrs[j], 20.0, 20);
    }
    handle = cmb_event_pattern_find(test_action, (void *)evstrs[2], (void *)evstrs[0]);
    (void)cmb_event_reschedule(handle, cmb_time() + 25.0);
    handle = cmb_event_pattern_find(test_action, (void *)evstrs[2], (void *)evstrs[1]);
    (void)cmb_event_reprioritize(handle, 3);

    r->counter[4] = cmb_event_pattern_count(CMB_ANY_ACTION, evstrs[1], CMB_ANY_OBJECT);
    r->counter[5] = cmb_event_pattern_cancel(CMB_ANY_ACTION, evstrs[1], CMB_ANY_OBJECT);
    r->counter[6] = cmb_event_queue_count();

    cmb_event_queue_execute();
    r->events = g_pops;
    r->t_end = cmb_time();
    r->counter[7] = g_actions;
    cmb_event_queue_terminate();
    cmb_random_terminate();
}

int event_ref_run_trials(uint64_t master_seed, uint64_t first, uint64_t count, uint64_t trace_cap, uint64_t *trace_key,
                         double *trace_time, struct event_result *out)
{
    for (uint64_t i = 0; i < count; i++) {
        run_event_trial(cmb_random_fmix64(master_seed, first + i), trace_cap, trace_cap ? trace_key + i * trace_cap : NULL,
                        trace_cap ? trace_time + i * trace_cap : NULL, &out[i]);
    }
    return 0;
}
