// examples/event_model.cuh - the event list used as a whole: cmb_event_queue_initialize / _is_empty / _count / _clear,
// cmb_event_time / _priority and cmb_event_pattern_find / _count / _cancel with the CMB_ANY_* wildcards, on either engine.
//
// EventTestT is the reference's own test of its event queue (test/test_event.c, test_events()) as model code: the queue starts
// at time 3, nine test_action events (subjects and objects foo, bar, yuk = 0, 1, 2) and an end_sim at 100 are scheduled, one is
// found and cancelled, every test_action of subject yuk is found and cancelled one by one, three more go in at t = 20, p = 20,
// one is rescheduled and one reprioritized, the events of subject bar are counted and cancelled, and the rest runs until end_sim
// clears the queue; every test_action reschedules itself.  NULL is cmb::NIL.  Its row:
//   counters[0] the handle the first pattern_find returned     [1] the bits of that event's cmb_event_time   [2] its priority
//   counters[3] the handles the wildcard loop cancelled, 16 bits each, the first in the low bits
//   counters[4] the pattern_count result   [5] the pattern_cancel result   [6] cmb_event_queue_count() before the run
//   counters[7] test_action events executed
// The pop trace carries the order the events ran in.  On the static tier the wildcard loop's first find has three matches,
// whose order is the general engine's heap array: every trial is flagged there and re-run on the general engine.
//
// EventChurnT is a model the static tier answers exactly: three processes hold exponential times while four tickers (events of
// subjects 0..3) reschedule themselves.  Each tick queries the list's count and emptiness, counts the blips (short events) of its
// group and the events of another ticker's subject, finds the next ticker (the only event that can match), reads its time and
// priority and reschedules it, cancels its group's blips once there are two, and adds a blip.  An end event at num_objects
// clears the queue.  Its row:
//   counters[0] sum of cmb_event_queue_count() at every event   [1] times cmb_event_queue_is_empty() was true
//   counters[2] sum of the bits of the found tickers' times      [3] sum of their priorities
//   counters[4] sum of the blip counts + 1000 x the counts by another ticker's subject (processes 0..2 never match)
//   counters[5] xor of the found handles   [6] blips cancelled by pattern   [7] ticks and blips executed
//   objects     process wake-ups
#pragma once

#include "../cimba_b200/csrc/cmb_static.cuh"

namespace event_example {
using namespace cimba_b200;

// What EventTestT reports as it goes, so that a printer of the reference's text (test code) can follow it; on the device, nothing.
enum : uint32_t {
    NOTE_START,         // after cmb_event_queue_initialize: t = the clock
    NOTE_SCHEDULED,     // a = the handle of one of the nine
    NOTE_QUEUE,         // a = which of the reference's cmb_event_queue_print calls (0..6 before the run)
    NOTE_FOUND,         // a = the handle, t = its time, p = its priority
    NOTE_CANCELING,     // a = a handle the wildcard loop cancels
    NOTE_COUNTED,       // a = the pattern_count result
    NOTE_CANCELLED,     // a = the pattern_cancel result
    NOTE_EXECUTE,       // the end of run_trial: t = the clock
    NOTE_ACTION,        // an event runs: a = the action, p = the subject, t = the object
};

struct NoNote {
    template <class S>
    static CMB_FN void at(S &, uint32_t, uint64_t, double, int64_t) {}
};

template <class S, class Note = NoNote>
struct EventTestT {
    enum : uint32_t { TEST_ACTION = cmb::ACT_CMB_USER, END_SIM };
    enum : uint32_t { FOO = 0u, BAR = 1u, YUK = 2u };
    static constexpr bool static_interrupts = true;     // the tier's second form ...
    static constexpr bool static_waits = true;          // ... with events by handle
    uint64_t counter[8];

    CMB_FN void process(S &, uint32_t, uint32_t, int64_t) {}
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    // test_action prints a line and reschedules itself; end_sim clears the queue
    CMB_FN void event(S &sim, uint32_t act, uint32_t subj, int64_t obj)
    {
        Note::at(sim, NOTE_ACTION, act, (double)obj, (int64_t)subj);
        if (act == TEST_ACTION) {
            counter[7]++;
            // the reference's call evaluates its arguments right to left (gcc, x86-64): the priority is drawn first
            const int64_t p = (int16_t)cmb_random_dice(1, 5);
            const double t = __dadd_rn(cmb_time(), cmb_random_exponential(10.0));
            (void)cmb_event_schedule(TEST_ACTION, subj, obj, t, p);
        }
        else {
            cmb_event_queue_clear();
        }
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &)
    {
        for (int k = 0; k < 8; k++) counter[k] = 0u;
        cmb_event_queue_initialize(3.0);
        Note::at(sim, NOTE_START, 0u, cmb_time(), 0);
        for (uint32_t i = 0u; i < 3u; i++) {
            for (uint32_t j = 0u; j < 3u; j++) {
                const double t = __dadd_rn(cmb_time(), cmb_random_exponential(10.0));
                const int64_t p = cmb_random_dice(1, 5);
                const uint64_t h = cmb_event_schedule(TEST_ACTION, i, j, t, p);
                Note::at(sim, NOTE_SCHEDULED, h, t, p);
            }
        }
        (void)cmb_event_schedule(END_SIM, cmb::NIL, cmb::NIL, 100.0, 0);
        Note::at(sim, NOTE_QUEUE, 0u, 0.0, 0);

        uint64_t h = cmb_event_pattern_find(TEST_ACTION, BAR, FOO);
        const double ht = cmb_event_time(h);
        const int64_t hp = cmb_event_priority(h);
        counter[0] = h;
        counter[1] = (uint64_t)__double_as_longlong(ht);
        counter[2] = (uint64_t)hp;
        Note::at(sim, NOTE_FOUND, h, ht, hp);
        (void)cmb_event_cancel(h);
        (void)cmb_event_pattern_find(TEST_ACTION, BAR, FOO);
        Note::at(sim, NOTE_QUEUE, 1u, 0.0, 0);

        for (uint32_t n = 0u; (h = cmb_event_pattern_find(TEST_ACTION, YUK, CMB_ANY_OBJECT)) != 0u; n++) {
            Note::at(sim, NOTE_CANCELING, h, 0.0, 0);
            if (n < 4u) counter[3] |= (h & 0xffffu) << (16u * n);
            (void)cmb_event_cancel(h);
        }
        Note::at(sim, NOTE_QUEUE, 2u, 0.0, 0);

        for (uint32_t j = 0u; j < 3u; j++) (void)cmb_event_schedule(TEST_ACTION, YUK, j, 20.0, 20);
        Note::at(sim, NOTE_QUEUE, 3u, 0.0, 0);

        h = cmb_event_pattern_find(TEST_ACTION, YUK, FOO);
        (void)cmb_event_reschedule(h, __dadd_rn(cmb_time(), 25.0));
        h = cmb_event_pattern_find(TEST_ACTION, YUK, BAR);
        (void)cmb_event_reprioritize(h, 3);
        Note::at(sim, NOTE_QUEUE, 4u, 0.0, 0);

        counter[4] = cmb_event_pattern_count(CMB_ANY_ACTION, BAR, CMB_ANY_OBJECT);
        Note::at(sim, NOTE_COUNTED, counter[4], 0.0, 0);
        Note::at(sim, NOTE_QUEUE, 5u, 0.0, 0);
        counter[5] = cmb_event_pattern_cancel(CMB_ANY_ACTION, BAR, CMB_ANY_OBJECT);
        Note::at(sim, NOTE_CANCELLED, counter[5], 0.0, 0);
        Note::at(sim, NOTE_QUEUE, 6u, 0.0, 0);

        counter[6] = cmb_event_queue_count();
        Note::at(sim, NOTE_EXECUTE, 0u, cmb_time(), 0);
    }

    CMB_FN void finish(S &, cmb::TrialOut &out)
    {
        out.objects = 0u;
        out.sum_wait = 0.0;
        out.max_queue = 0u;
        for (int k = 0; k < 8; k++) out.counters[k] = counter[k];
    }
};

template <class S>
struct EventChurnT {
    enum : uint32_t { TICK = cmb::ACT_CMB_USER, BLIP, END };
    static constexpr uint32_t PROCS = 3u, TICKERS = 4u, GROUP0 = 10u;
    static constexpr bool static_interrupts = true;
    static constexpr bool static_waits = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t) { return 0u; }
    uint64_t counter[8];
    uint64_t wakeups;
    double   hold_mean;

    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void process(S &sim, uint32_t me, uint32_t, int64_t sig)
    {
        EventChurnT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(hold_mean);
            wakeups++;
            counter[0] += cmb_event_queue_count();
        }
        CMB_PROCESS_END
    }

    CMB_FN void event(S &sim, uint32_t act, uint32_t subj, int64_t obj)
    {
        counter[0] += cmb_event_queue_count();
        if (act == END) {
            cmb_event_queue_clear();
            counter[1] += cmb_event_queue_is_empty() ? 1u : 0u;
            return;
        }
        counter[7]++;
        if (act == BLIP) return;
        counter[1] += cmb_event_queue_is_empty() ? 1u : 0u;
        const uint32_t group = GROUP0 + (subj & 1u);
        const uint64_t blips = cmb_event_pattern_count(BLIP, group, CMB_ANY_OBJECT);
        counter[4] += blips + 1000u * cmb_event_pattern_count(CMB_ANY_ACTION, (subj + 2u) % TICKERS, CMB_ANY_OBJECT);
        const uint64_t next = cmb_event_pattern_find(TICK, (subj + 1u) % TICKERS, CMB_ANY_OBJECT);
        counter[5] ^= next;
        counter[2] += (uint64_t)__double_as_longlong(cmb_event_time(next));
        counter[3] += (uint64_t)cmb_event_priority(next);
        const double moved = __dadd_rn(cmb_time(), cmb_random_exponential(2.0));
        (void)cmb_event_reschedule(next, moved);
        if (blips >= 2u) counter[6] += cmb_event_pattern_cancel(CMB_ANY_ACTION, group, CMB_ANY_OBJECT);
        const double tb = __dadd_rn(cmb_time(), cmb_random_exponential(1.5));
        const int64_t pb = cmb_random_dice(-2, 2);
        (void)cmb_event_schedule(BLIP, group, obj, tb, pb);
        const double tt = __dadd_rn(cmb_time(), cmb_random_exponential(1.0));
        const int64_t pt = cmb_random_dice(1, 3);
        (void)cmb_event_schedule(TICK, subj, obj + 1, tt, pt);
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        for (int k = 0; k < 8; k++) counter[k] = 0u;
        wakeups = 0u;
        hold_mean = in.srv_mean;
        for (uint32_t i = 0u; i < PROCS; i++) cmb_process_start(cmb_process_create(0u, 0, i));
        for (uint32_t s = 0u; s < TICKERS; s++) {
            const double t = cmb_random_exponential(1.0);
            const int64_t p = cmb_random_dice(1, 3);
            (void)cmb_event_schedule(TICK, s, 0, t, p);
        }
        (void)cmb_event_schedule(END, cmb::NIL, cmb::NIL, (double)in.num_objects, 0);
    }

    CMB_FN void finish(S &, cmb::TrialOut &out)
    {
        out.objects = wakeups;
        out.sum_wait = 0.0;
        out.max_queue = 0u;
        for (int k = 0; k < 8; k++) out.counters[k] = counter[k];
    }
};

// the pending events of its own each model can have at once on the static tier: EventTestT ten (nine and end_sim), EventChurnT
// nine (four tickers, two blips per group, the end event) - one to spare
constexpr int EVENT_TEST_SLOTS = 10;
constexpr int EVENT_CHURN_SLOTS = 10;

template <class S>
using EventTest = EventTestT<S>;

}  // namespace event_example
