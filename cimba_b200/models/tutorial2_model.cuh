// tutorial2_model.cuh - the reference's second tutorial, tutorial/tut_2_1.c, written against the authoring surface: five mice that
// set themselves a random priority and acquire 1..5 units of a 20-unit cmb_resourcepool, two rats that PRE-EMPT 3..10 units, a cat
// that interrupts a random rodent with CMB_PROCESS_INTERRUPTED or a signal of its own (cmb_random_flip decides which, and whether
// it strikes again), everybody holding and partly releasing in between; an end event at t = 100 000 stops all eight.
// (test/test_resourcepool.c is a variant of it with other numbers: cheese_model.cuh.)
// Oracle: the UNMODIFIED tutorial source as a program, one fresh process per trial (oracle/ref_build/tut2_main.c ->
// oracle/_ref/tut2_ref): the pool breaks priority ties by process address - creation order in a fresh process, which is what the
// index-based key gives here (SURVEY.md quirk 4) - and cmb_random_flip's cached bits outlive a trial.
//   counters[0] = the random stream's next raw output after the run (a fingerprint of every draw), [1] = units in use at the end,
//   [2] = successful acquires + pre-empts; objects = the same.
// A template over the engine, as tutorial1_model.cuh: cmb::Sim, or the static tier's second form (static_interrupts).
#pragma once
#include "../csrc/cmb_kernel.cuh"
#include "../csrc/cmb_static.cuh"

namespace cimba_b200 {
namespace models {

template <class S>
struct Tutorial2T {
    typename S::resourcepool_type cheese;
    uint64_t successes;
    enum : uint32_t { MOUSE, RAT, CAT };
    enum : uint32_t { END_SIM = cmb::ACT_CMB_USER };
    static constexpr uint32_t MICE = 5u, RATS = 2u, CATS = 1u, RODENTS = 7u;
    static constexpr bool static_interrupts = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i < MICE ? MOUSE : (i < RODENTS ? RAT : CAT); }
    template <class F>
    CMB_FN void static_holdables(F &&visit) { visit(cheese); }

    // mousefunc :59-127 / ratfunc :129-197; u[0] = amount_held, u[1] = the amount of the call in progress
    CMB_FN void rodent(S &sim, uint32_t me, int64_t sig, bool rat)
    {
        Tutorial2T &m = *this;
        CMB_PROCESS_BEGIN
        sim.proc[me].u[0] = 0u;
        for (;;) {
            if (rat) {
                sim.proc[me].u[1] = (uint64_t)cmb_random_dice(3, 10);
                cmb_process_priority_set(me, cmb_random_dice(-5, 15));
                CMB_RESOURCEPOOL_PREEMPT(cheese, sim.proc[me].u[1]);
            }
            else {
                sim.proc[me].u[1] = (uint64_t)cmb_random_dice(1, 5);
                cmb_process_priority_set(me, cmb_random_dice(-10, 10));
                CMB_RESOURCEPOOL_ACQUIRE(cheese, sim.proc[me].u[1]);
            }
            if (sig == CMB_PROCESS_SUCCESS) {
                sim.proc[me].u[0] += sim.proc[me].u[1];
                successes += 1u;
            }
            else if (sig == CMB_PROCESS_PREEMPTED) {
                sim.proc[me].u[0] = 0u;
            }
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            if (sig == CMB_PROCESS_PREEMPTED) sim.proc[me].u[0] = 0u;
            if (sim.proc[me].u[0] > 1u) {
                sim.proc[me].u[1] = (uint64_t)cmb_random_dice(1, (long long)sim.proc[me].u[0]);
                CMB_RESOURCEPOOL_RELEASE(cheese, sim.proc[me].u[1]);
                sim.proc[me].u[0] -= sim.proc[me].u[1];
            }
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            if (sig == CMB_PROCESS_PREEMPTED) sim.proc[me].u[0] = 0u;
        }
        CMB_PROCESS_END
    }

    CMB_FN void cat(S &sim, uint32_t me, int64_t sig)                    // catfunc, :199-224
    {
        Tutorial2T &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(5.0);
            do {
                CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
                pounce(sim);
            } while (cmb_random_flip());
        }
        CMB_PROCESS_END
    }

    CMB_FN void pounce(S &sim)
    {
        const uint32_t target = (uint32_t)cmb_random_dice(0, (long long)RODENTS - 1);
        const int64_t with = cmb_random_flip() ? CMB_PROCESS_INTERRUPTED : (int64_t)cmb_random_dice(10, 100);
        cmb_process_interrupt(target, with, 0);
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &)                  // :226-271
    {
        successes = 0u;
        cmb_resourcepool_initialize(cheese, 20u);
        for (uint32_t i = 0u; i < RODENTS + CATS; i++) {
            const int64_t pri = cmb_random_dice(-5, 5);
            cmb_process_start(cmb_process_create(i < MICE ? MOUSE : (i < RODENTS ? RAT : CAT), pri, i));
        }
        (void)cmb_event_schedule(END_SIM, cmb::NIL, 0, 100000.0, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == CAT) cat(sim, me, sig);
        else rodent(sim, me, sig, kind == RAT);
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)       // end_sim_evt, :40-57
    {
        Tutorial2T &m = *this;
        if (action == END_SIM) {
            for (uint32_t i = 0u; i < RODENTS + CATS; i++) cmb_process_stop(i, 0);
        }
    }
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        out.counters[0] = sim.rng.next();
        out.counters[1] = cmb_resourcepool_in_use(cheese);
        out.counters[2] = successes;
        out.objects = successes;
        out.sum_wait = 0.0;
    }
};

using Tutorial2 = Tutorial2T<cmb::Sim>; // on the static tier: Tutorial2T<cmb::StaticSimOf<Tutorial2T, 8, 0, 8>> (eight processes, eight spare event slots)

}  // namespace models
}  // namespace cimba_b200
