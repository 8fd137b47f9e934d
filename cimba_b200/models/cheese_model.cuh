// cheese_model.cuh - the reference's own pool test, test/test_resourcepool.c:50-305, as it stands, written against the
// authoring surface: three mice (cmb_process_priority_set + cmb_resourcepool_acquire of 1..10 units), two rats
// (cmb_resourcepool_preempt), a cat interrupting a random rodent (cmb_random_flip picks INTERRUPTED or a signal in 10..100),
// the pool's usage history on, an end event that stops everybody.  With 20 units, 100 time units and the reference's seed
// it reproduces test/reference/resourcepool.txt ("N 120  Mean 19.77  StdDev 1.147  ...") - the golden file that depends
// on the holders' tie-break by process address (SURVEY.md quirk 4): the test creates its processes one after the other, so
// address order is creation order, which is what the index-based key (pid + 1) gives.
// Oracle: the same test against the reference's API, oracle/ref_build/ref_driver.c model 18.
// A template over the engine, as tutorial1_model.cuh: cmb::Sim, or the static tier's second form (static_interrupts: priorities,
// interrupts, pre-emption; the pool named in static_holdables, so that the end event's stops drop the holdings there).
#pragma once
#include "../csrc/cmb_kernel.cuh"
#include "../csrc/cmb_static.cuh"

namespace cimba_b200 {
namespace models {

template <class S>
struct CheeseT {
    typename S::recorded_resourcepool_type cheese;
    uint64_t successes;
    double   sum_time;
    enum : uint32_t { MOUSE, RAT, CAT };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER };
    static constexpr uint32_t MICE = 3u, RATS = 2u, RODENTS = 5u;
    static constexpr bool static_interrupts = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i < MICE ? MOUSE : (i < RODENTS ? RAT : CAT); }
    template <class F>
    CMB_FN void static_holdables(F &&visit) { visit(cheese); }

    // one rodent: u[0] = amount held (the body's local), u[1] = the amount of the call in progress
    CMB_FN void rodent(S &sim, uint32_t me, int64_t sig, bool rat)
    {
        CheeseT &m = *this;
        CMB_PROCESS_BEGIN
        sim.proc[me].u[0] = 0u;
        for (;;) {
            sim.proc[me].u[1] = (uint64_t)cmb_random_dice(1, 10);
            if (rat) {
                CMB_RESOURCEPOOL_PREEMPT(cheese, sim.proc[me].u[1]);
            }
            else {
                cmb_process_priority_set(me, cmb_random_dice(-10, 10));
                CMB_RESOURCEPOOL_ACQUIRE(cheese, sim.proc[me].u[1]);
            }
            if (sig == CMB_PROCESS_SUCCESS) {
                sim.proc[me].u[0] += sim.proc[me].u[1];
                successes += 1u;
                sum_time += cmb_time();
                CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
                if (sig == CMB_PROCESS_SUCCESS) {
                    uint64_t rel = (uint64_t)cmb_random_dice(1, 10);
                    if (rel > sim.proc[me].u[0]) rel = sim.proc[me].u[0];
                    CMB_RESOURCEPOOL_RELEASE(cheese, rel);
                    sim.proc[me].u[0] -= rel;
                }
                else if (sig == CMB_PROCESS_PREEMPTED) {
                    sim.proc[me].u[0] = 0u;
                }
            }
            else if (sig == CMB_PROCESS_PREEMPTED) {
                sim.proc[me].u[0] = 0u;
            }
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            if (sig == CMB_PROCESS_PREEMPTED) sim.proc[me].u[0] = 0u;
        }
        CMB_PROCESS_END
    }

    CMB_FN void cat(S &sim, uint32_t me, int64_t sig)
    {
        CheeseT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            {
                const uint32_t victim = (uint32_t)cmb_random_dice(0, (long long)RODENTS - 1);
                const int64_t loud = cmb_random_dice(10, 100);
                cmb_process_interrupt(victim, cmb_random_flip() ? CMB_PROCESS_INTERRUPTED : loud, 0);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)                // test_pool, :307-379
    {
        successes = 0u;
        sum_time = 0.0;
        cmb_resourcepool_initialize(cheese, (uint64_t)in.servers);
        cmb_resourcepool_start_recording(cheese);
        for (uint32_t i = 0u; i <= RODENTS; i++) {
            const int64_t pri = cmb_random_dice(-5, 5);
            cmb_process_start(cmb_process_create(i < MICE ? MOUSE : (i < RODENTS ? RAT : CAT), pri, i));
        }
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == CAT) cat(sim, me, sig);
        else rodent(sim, me, sig, kind == RAT);
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)       // end_sim_evt, :50-72
    {
        CheeseT &m = *this;
        if (action == END_EVENT) {
            for (uint32_t i = 0u; i <= RODENTS; i++) cmb_process_stop(i, 0);
        }
    }
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        cmb_resourcepool_stop_recording(cheese);
        const cmb_wtdsummary &h = cheese.history.acc;   // what cmb_timeseries_summarize makes of the stored history
        cmb_summary_to_counters(out, &h);
        out.objects = successes;
        out.sum_wait = sum_time;
        out.max_queue = (uint32_t)h.count;
    }
};

using Cheese = CheeseT<cmb::Sim>;       // on the static tier: CheeseT<cmb::StaticSimOf<CheeseT, 6, 0, 6>> (six processes, six spare event slots)

}  // namespace models
}  // namespace cimba_b200
