// coverage_models.cuh - the three "everything at once" workloads of the parity suite written against the authoring surface
// (the same worlds the reference runs in oracle/ref_build/ref_driver.c, where the counters are described):
//   PoolFightT    (model 4) test/test_resourcepool.c's cast with checks: mice changing their own priority and acquiring, rats
//                 pre-empting, a cat interrupting, partial releases, cmb_resourcepool_held_by_process compared with the body's own count
//   QueueAndTideT (model 6) cmb_priorityqueue put / get / position / cancel / reprioritize by handle + cmb_condition with two
//                 predicates, under a nuisance
//   FrontDeskT    (model 8) timers (add / cancel / set / clear), cmb_process_yield + resume, wait_process on a process that exits
//                 and is started again, wait_event on events that get rescheduled / reprioritized / cancelled, a condition whose
//                 guard OBSERVES a resource's guard
// Each is a template over the engine (cmb::Sim, or the static tier's second form); PoolFight, QueueAndTide and FrontDesk name their
// general-engine forms.
#pragma once
#include "../csrc/cmb_kernel.cuh"
#include "../csrc/cmb_static.cuh"

namespace cimba_b200 {
namespace models {

// A template over the engine: PoolFightT<cmb::Sim> is the general-engine model (PoolFight); on the static tier it runs in the
// second form with 6 processes and POOLFIGHT_SPARE_SLOTS spare event slots for the end event, the cat's interrupt and a rat's
// pre-emption, which interrupts every victim at once.  4 is the fewest at which no vector case of
// tests/golden/cmb_engine_vectors.json flags (with 3, half of them do); a trial that needs more is flagged and re-run on the general
// engine - about 1.9 % of them at capacity 10 and 500 time units.
constexpr int POOLFIGHT_SPARE_SLOTS = 4;

template <class S>
struct PoolFightT {
    typename S::resourcepool_type pool;
    uint64_t counter[8];
    double   sum_wait;
    enum : uint32_t { MOUSE, RAT, CAT };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER };
    static constexpr uint32_t MICE = 3u, RODENTS = 5u;
    static constexpr bool static_interrupts = true;
    static constexpr bool static_fel_high = true;
    static constexpr int static_min_ctas = 1;       // without it ptxas holds the kernel to 128 registers and spills
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i < MICE ? MOUSE : i < RODENTS ? RAT : CAT; }
    template <class F>
    CMB_FN void static_holdables(F &&visit) { visit(pool); }

    CMB_FN void check(S &sim, uint32_t me)
    {
        if (cmb_resourcepool_held_by_process(pool, me) != sim.proc[me].u[0]) counter[7] += 1u;
    }

    CMB_FN void signal(S &sim, uint32_t me, int64_t sig)
    {
        if (sig == CMB_PROCESS_PREEMPTED) {
            counter[2] += 1u;
            sim.proc[me].u[0] = 0u;
        }
        else if (sig != CMB_PROCESS_SUCCESS) {
            counter[3] += 1u;
        }
        counter[4] += (uint64_t)sig;
    }

    // u[0] = units held by the body's own count, u[1] = the request in progress
    CMB_FN void rodent(S &sim, uint32_t me, int64_t sig, bool rat)
    {
        PoolFightT &m = *this;
        CMB_PROCESS_BEGIN
        sim.proc[me].u[0] = 0u;
        for (;;) {
            check(sim, me);
            sim.proc[me].u[1] = (uint64_t)cmb_random_dice(1, 5);
            if (rat) {
                CMB_RESOURCEPOOL_PREEMPT(pool, sim.proc[me].u[1]);
            }
            else {
                cmb_process_priority_set(me, cmb_random_dice(-5, 5));
                CMB_RESOURCEPOOL_ACQUIRE(pool, sim.proc[me].u[1]);
            }
            if (sig == CMB_PROCESS_SUCCESS) {
                sim.proc[me].u[0] += sim.proc[me].u[1];
                counter[rat ? 1 : 0] += 1u;
                check(sim, me);
                CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
                if (sig == CMB_PROCESS_SUCCESS) {
                    uint64_t rel = (uint64_t)cmb_random_dice(1, 5);
                    if (rel > sim.proc[me].u[0] || cmb_random_dice(0, 1) == 1) rel = sim.proc[me].u[0];
                    CMB_RESOURCEPOOL_RELEASE(pool, rel);
                    sim.proc[me].u[0] -= rel;
                    counter[5] += rel;
                    sum_wait = __dadd_rn(sum_wait, __dmul_rn(cmb_time(), (double)rel));
                }
                else {
                    signal(sim, me, sig);
                }
            }
            else {
                signal(sim, me, sig);
            }
            check(sim, me);
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            if (sig != CMB_PROCESS_SUCCESS) signal(sim, me, sig);
        }
        CMB_PROCESS_END
    }

    CMB_FN void cat(S &sim, uint32_t me, int64_t sig)
    {
        PoolFightT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            {
                const uint32_t victim = (uint32_t)cmb_random_dice(0, (long long)RODENTS - 1);
                const int64_t loud = cmb_random_dice(10, 100);
                cmb_process_interrupt(victim, cmb_random_dice(0, 1) == 1 ? CMB_PROCESS_INTERRUPTED : loud, 0);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        for (uint32_t i = 0u; i < 8u; i++) counter[i] = 0u;
        sum_wait = 0.0;
        cmb_resourcepool_initialize(pool, (uint64_t)in.servers);
        for (uint32_t i = 0u; i < RODENTS; i++) {
            const int64_t pri = cmb_random_dice(-5, 5);
            cmb_process_start(cmb_process_create(i < MICE ? MOUSE : RAT, pri, i));
        }
        cmb_process_start(cmb_process_create(CAT, 0, RODENTS));
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == CAT) cat(sim, me, sig);
        else rodent(sim, me, sig, kind == RAT);
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)
    {
        PoolFightT &m = *this;
        if (action == END_EVENT) {
            for (uint32_t i = 0u; i <= RODENTS; i++) cmb_process_stop(i, 0);
        }
    }
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        counter[6] = cmb_resourcepool_in_use(pool);
        for (uint32_t i = 0u; i < 8u; i++) out.counters[i] = counter[i];
        out.objects = counter[0] + counter[1];
        out.sum_wait = sum_wait;
        out.max_queue = sim.fel_high;
    }
};

using PoolFight = PoolFightT<cmb::Sim>;

// A template over the engine: QueueAndTideT<cmb::Sim> is the general-engine model (QueueAndTide); on the static tier it runs in the
// second form with 8 processes and 2 spare event slots (the end event and the nuisance's interrupt), its priority queue in the
// tier's table and the condition's wake-ups in the waiters' own slots.
template <class S>
struct QueueAndTideT {
    typename S::priorityqueue_type pq;
    typename S::condition_type     tide_cv;
    uint64_t counter[8];
    uint64_t last_handle[2];
    double   sum_wait, put_mean, get_mean;
    long long level, threshold[2];
    enum : uint32_t { PRODUCER, CONSUMER, SHUFFLER, TIDE, WAITER, NUISANCE };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER };
    enum : uint32_t { HIGH_ENOUGH = 100u };
    static constexpr uint32_t PROCS = 7u;
    static constexpr bool static_interrupts = true;
    static constexpr bool static_fel_high = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i)
    {
        return i < 2u ? PRODUCER : i == 2u ? CONSUMER : i == 3u ? SHUFFLER : i == 4u ? TIDE : i < PROCS ? WAITER : NUISANCE;
    }

    CMB_FN void note(int64_t sig)
    {
        if (sig != CMB_PROCESS_SUCCESS) counter[6] += (uint64_t)sig;
    }

    // u[0] = weight, u[1] = handle, fr... the priority of the put lives in proc.f[0] (as an integer value)
    CMB_FN void producer(S &sim, uint32_t me, int64_t sig)
    {
        QueueAndTideT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(put_mean);
            note(sig);
            sim.proc[me].u[0] = (uint64_t)cmb_random_dice(1, 9);
            sim.proc[me].f[0] = (double)cmb_random_dice(-3, 3);
            sim.proc[me].u[1] = 0u;
            CMB_PRIORITYQUEUE_PUT(pq, sim.proc[me].u[0], (int64_t)sim.proc[me].f[0], &sim.proc[me].u[1]);
            if (sig == CMB_PROCESS_SUCCESS) {
                counter[0] += 1u;
                last_handle[me] = sim.proc[me].u[1];
            }
            else {
                counter[2] += 1u;
                note(sig);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void consumer(S &sim, uint32_t me, int64_t sig)
    {
        QueueAndTideT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(get_mean);
            note(sig);
            CMB_PRIORITYQUEUE_GET(pq, sim.proc[me].u[0]);
            if (sig == CMB_PROCESS_SUCCESS) {
                counter[1] += sim.proc[me].u[0];
                sum_wait = __dadd_rn(sum_wait, __dmul_rn(cmb_time(), (double)sim.proc[me].u[0]));
            }
            else {
                counter[2] += 1u;
                note(sig);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void shuffler(S &sim, uint32_t me, int64_t sig)
    {
        QueueAndTideT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(1.5);
            note(sig);
            {
                const uint64_t handle = last_handle[cmb_random_dice(0, 1)];
                if (handle != 0u) {
                    const uint64_t pos = cmb_priorityqueue_position(pq, handle);
                    counter[3] += pos;
                    if (pos > 0u) {
                        if (cmb_random_dice(0, 1) == 1) {
                            cmb_priorityqueue_reprioritize(pq, handle, cmb_random_dice(-3, 3));
                        }
                        else {
                            (void)cmb_priorityqueue_cancel(pq, handle);
                            counter[3] += 1000u;
                        }
                    }
                }
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void tide(S &sim, uint32_t me, int64_t sig)
    {
        QueueAndTideT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            note(sig);
            level = cmb_random_dice(0, 5);
            counter[4] += cmb_condition_signal(tide_cv);
        }
        CMB_PROCESS_END
    }

    // u[0] = "through" flag of the pass in progress
    CMB_FN void waiter(S &sim, uint32_t me, int64_t sig)
    {
        QueueAndTideT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            sim.proc[me].u[0] = 1u;
            while (level < threshold[me - 5u]) {
                CMB_CONDITION_WAIT(tide_cv, HIGH_ENOUGH, (int32_t)(me - 5u));
                if (sig != CMB_PROCESS_SUCCESS) {
                    note(sig);
                    sim.proc[me].u[0] = 0u;
                    break;
                }
            }
            if (sim.proc[me].u[0]) counter[5] += 1u;
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            note(sig);
        }
        CMB_PROCESS_END
    }

    CMB_FN void nuisance(S &sim, uint32_t me, int64_t sig)
    {
        QueueAndTideT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            {
                const uint32_t victim = (uint32_t)cmb_random_dice(0, (long long)PROCS - 1);
                const int64_t loud = cmb_random_dice(1, 10);
                const int64_t pri = cmb_random_dice(-5, 5);
                cmb_process_interrupt(victim, loud, pri);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        for (uint32_t i = 0u; i < 8u; i++) counter[i] = 0u;
        sum_wait = 0.0;
        put_mean = in.arr_mean;
        get_mean = in.srv_mean;
        last_handle[0] = last_handle[1] = 0u;
        level = 0;
        threshold[0] = 2;
        threshold[1] = 4;
        cmb_priorityqueue_initialize(pq, (uint64_t)in.servers);
        cmb_condition_initialize(tide_cv);
        const uint32_t kind[PROCS] = { PRODUCER, PRODUCER, CONSUMER, SHUFFLER, TIDE, WAITER, WAITER };
        for (uint32_t i = 0u; i < PROCS; i++) {
            const int64_t pri = cmb_random_dice(-5, 5);
            cmb_process_start(cmb_process_create(kind[i], pri, i));
        }
        cmb_process_start(cmb_process_create(NUISANCE, 0, PROCS));
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        switch (kind) {
        case PRODUCER: producer(sim, me, sig); break;
        case CONSUMER: consumer(sim, me, sig); break;
        case SHUFFLER: shuffler(sim, me, sig); break;
        case TIDE:     tide(sim, me, sig); break;
        case WAITER:   waiter(sim, me, sig); break;
        default:       nuisance(sim, me, sig); break;
        }
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)
    {
        QueueAndTideT &m = *this;
        if (action == END_EVENT) {
            for (uint32_t i = 0u; i <= PROCS; i++) cmb_process_stop(i, 0);
        }
    }

    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t ctx) { return level >= threshold[ctx]; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        counter[7] = cmb_priorityqueue_length(pq);
        for (uint32_t i = 0u; i < 8u; i++) out.counters[i] = counter[i];
        out.objects = counter[0];
        out.sum_wait = sum_wait;
        out.max_queue = sim.fel_high;
    }
};

using QueueAndTide = QueueAndTideT<cmb::Sim>;

// A template over the engine: FrontDeskT<cmb::Sim> is the general-engine model (FrontDesk); on the static tier it runs in the
// second form with static_waits - 8 processes and FRONTDESK_SPARE_SLOTS spare event slots for the end event, the bells, the
// patients' timers, the nuisance's interrupt, the clerk's resumes and the wake-ups of waits on the clerk and on the bell.
// 8 is the most the vector cases of tests/golden/cmb_engine_vectors.json have pending at once: with 7 some of them flag, with 8
// none.  A trial that needs more is flagged and re-run on the general engine.
constexpr int FRONTDESK_SPARE_SLOTS = 8;

template <class S>
struct FrontDeskT {
    typename S::resource_type  desk;
    typename S::condition_type desk_free;
    uint64_t counter[8];
    uint64_t bell;
    double   sum_wait, arr_mean, srv_mean;
    uint32_t clerk_start_pending;
    enum : uint32_t { PATIENT, CLERK, SUPERVISOR, RINGER, LISTENER, WATCHER, NUISANCE };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER, BELL_EVENT };
    enum : uint32_t { DESK_IS_FREE = 100u };
    enum : int64_t { SIG_ALARM = 77, SIG_DOZE = 55, SIG_NUDGE = 9 };
    static constexpr uint32_t PROCS = 8u, THE_CLERK = 2u;
    static constexpr bool static_interrupts = true;
    static constexpr bool static_waits = true;
    static constexpr bool static_fel_high = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i)
    {
        return i < 2u ? PATIENT : i == 2u ? CLERK : i == 3u ? SUPERVISOR : i == 4u ? RINGER : i == 5u ? LISTENER : i == 6u ? WATCHER : NUISANCE;
    }
    template <class F>
    CMB_FN void static_holdables(F &&visit) { visit(desk); }

    CMB_FN void note(int64_t sig)
    {
        if (sig != CMB_PROCESS_SUCCESS) counter[7] += (uint64_t)sig;
    }

    // u[0] = the patience timer's handle, f[0] = when the desk was taken
    CMB_FN void patient(S &sim, uint32_t me, int64_t sig)
    {
        FrontDeskT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(arr_mean);
            note(sig);
            sim.proc[me].u[0] = cmb_process_timer_add(cmb_random_exponential(__dmul_rn(2.0, srv_mean)), CMB_PROCESS_TIMEOUT);
            CMB_RESOURCE_ACQUIRE(desk);
            if (sig == CMB_PROCESS_SUCCESS) {
                (void)cmb_process_timer_cancel(sim.proc[me].u[0]);
                counter[0] += 1u;
                sim.proc[me].f[0] = cmb_time();
                (void)cmb_process_timer_add(cmb_random_exponential(3.0), SIG_ALARM);
                CMB_PROCESS_HOLD_EXPONENTIAL(srv_mean);
                note(sig);
                cmb_process_timers_clear(me);
                CMB_RESOURCE_RELEASE(desk);
                sum_wait = __dadd_rn(sum_wait, __dsub_rn(cmb_time(), sim.proc[me].f[0]));
                cmb_process_timer_set(cmb_random_exponential(0.3), SIG_DOZE);
                CMB_PROCESS_YIELD();
                note(sig);
                if (sig != SIG_DOZE) cmb_process_timers_clear(me);
            }
            else if (sig == CMB_PROCESS_TIMEOUT) {
                counter[1] += 1u;
            }
            else {
                note(sig);
                cmb_process_timers_clear(me);
            }
        }
        CMB_PROCESS_END
    }

    // u[0] = jobs this time, u[1] = jobs done
    CMB_FN void clerk(S &sim, uint32_t me, int64_t sig)
    {
        FrontDeskT &m = *this;
        CMB_PROCESS_BEGIN
        clerk_start_pending = 0u;
        sim.proc[me].u[0] = (uint64_t)cmb_random_dice(2, 5);
        for (sim.proc[me].u[1] = 0u; sim.proc[me].u[1] < sim.proc[me].u[0]; sim.proc[me].u[1]++) {
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            note(sig);
            if (cmb_random_dice(0, 2) == 0) cmb_process_resume((uint32_t)cmb_random_dice(0, 1), SIG_NUDGE);
            counter[3] += 1u;
        }
        CMB_PROCESS_EXIT((int64_t)sim.proc[me].u[0]);
        CMB_PROCESS_END
    }

    CMB_FN void supervisor(S &sim, uint32_t me, int64_t sig)
    {
        FrontDeskT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_WAIT_PROCESS(THE_CLERK);
            if (sig == CMB_PROCESS_SUCCESS) {
                counter[2] += 1u;
                CMB_PROCESS_HOLD_EXPONENTIAL(0.5);
                note(sig);
                if (cmb_process_status(THE_CLERK) == CMB_PROCESS_FINISHED && !clerk_start_pending) {
                    clerk_start_pending = 1u;
                    cmb_process_start(THE_CLERK);
                }
            }
            else {
                note(sig);
            }
        }
        CMB_PROCESS_END
    }

    // u[0] = the bell's handle
    CMB_FN void ringer(S &sim, uint32_t me, int64_t sig)
    {
        FrontDeskT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            sim.proc[me].f[0] = __dadd_rn(cmb_time(), cmb_random_exponential(2.0));
            sim.proc[me].u[0] = cmb_event_schedule(BELL_EVENT, cmb::NIL, 0, sim.proc[me].f[0], cmb_random_dice(-2, 2));
            bell = sim.proc[me].u[0];
            CMB_PROCESS_HOLD_EXPONENTIAL(0.7);
            note(sig);
            if (cmb_event_is_scheduled(sim.proc[me].u[0])) {
                const long long op = cmb_random_dice(0, 3);
                if (op == 0) {
                    (void)cmb_event_reschedule(sim.proc[me].u[0], __dadd_rn(cmb_time(), cmb_random_exponential(1.0)));
                    counter[5] += 1u;
                }
                else if (op == 1) {
                    (void)cmb_event_reprioritize(sim.proc[me].u[0], cmb_random_dice(-5, 5));
                    counter[5] += 100u;
                }
                else if (op == 2) {
                    (void)cmb_event_cancel(sim.proc[me].u[0]);
                    counter[5] += 10000u;
                }
            }
            if (cmb_event_is_scheduled(sim.proc[me].u[0])) {
                CMB_PROCESS_WAIT_EVENT(sim.proc[me].u[0]);
                note(sig);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void listener(S &sim, uint32_t me, int64_t sig)
    {
        FrontDeskT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            if (bell != 0u && cmb_event_is_scheduled(bell)) {
                CMB_PROCESS_WAIT_EVENT(bell);
                if (sig == CMB_PROCESS_SUCCESS) counter[6] += 1000u;
                else note(sig);
            }
            else {
                CMB_PROCESS_HOLD_EXPONENTIAL(0.5);
                note(sig);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void watcher(S &sim, uint32_t me, int64_t sig)
    {
        FrontDeskT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_CONDITION_WAIT(desk_free, DESK_IS_FREE, 0);
            if (sig == CMB_PROCESS_SUCCESS) counter[6] += 1u;
            else note(sig);
            CMB_PROCESS_HOLD_EXPONENTIAL(0.8);
            note(sig);
        }
        CMB_PROCESS_END
    }

    CMB_FN void nuisance(S &sim, uint32_t me, int64_t sig)
    {
        FrontDeskT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            {
                const uint32_t victim = (uint32_t)cmb_random_dice(0, (long long)PROCS - 2);
                const int64_t loud = cmb_random_dice(1, 10);
                const int64_t pri = cmb_random_dice(-5, 5);
                if (cmb_process_status(victim) == CMB_PROCESS_RUNNING) cmb_process_interrupt(victim, loud, pri);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        FrontDeskT &m = *this;
        for (uint32_t i = 0u; i < 8u; i++) counter[i] = 0u;
        sum_wait = 0.0;
        arr_mean = in.arr_mean;
        srv_mean = in.srv_mean;
        bell = 0u;
        clerk_start_pending = 0u;
        cmb_resource_initialize(desk);
        cmb_condition_initialize(desk_free);
        cmb_resourceguard_register(desk.guard, desk_free.guard);
        const uint32_t kind[PROCS] = { PATIENT, PATIENT, CLERK, SUPERVISOR, RINGER, LISTENER, WATCHER, NUISANCE };
        for (uint32_t i = 0u; i < PROCS; i++) {
            const int64_t pri = (i + 1u < PROCS) ? cmb_random_dice(-5, 5) : 0;
            cmb_process_start(cmb_process_create(kind[i], pri, i));
        }
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        switch (kind) {
        case PATIENT:    patient(sim, me, sig); break;
        case CLERK:      clerk(sim, me, sig); break;
        case SUPERVISOR: supervisor(sim, me, sig); break;
        case RINGER:     ringer(sim, me, sig); break;
        case LISTENER:   listener(sim, me, sig); break;
        case WATCHER:    watcher(sim, me, sig); break;
        default:         nuisance(sim, me, sig); break;
        }
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)
    {
        FrontDeskT &m = *this;
        if (action == BELL_EVENT) {
            counter[4] += 1u;
        }
        else if (action == END_EVENT) {
            for (uint32_t i = 0u; i < PROCS; i++) {
                if (cmb_process_status(i) == CMB_PROCESS_RUNNING) cmb_process_stop(i, 0);
            }
        }
    }

    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return desk.holder == cmb::NIL; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        for (uint32_t i = 0u; i < 8u; i++) out.counters[i] = counter[i];
        out.objects = counter[0];
        out.sum_wait = sum_wait;
        out.max_queue = sim.fel_high;
    }
};

using FrontDesk = FrontDeskT<cmb::Sim>;

}  // namespace models
}  // namespace cimba_b200
