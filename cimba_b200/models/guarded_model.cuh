// guarded_model.cuh - the reference's queue tests, test/test_objectqueue.c:40-200 and test/test_priorityqueue.c, written
// against the authoring surface: three putters and three getters with random priorities on a BOUNDED queue (both guards in
// play), a nuisance process interrupting a random one of them with a random signal and event priority, an end event that
// stops all seven.  PRIORITY = false: a cmb_objectqueue (models 3 and, with the length history on, 11 - the golden file
// test/reference/objectqueue.txt); RECORD = the length history on; PRIORITY = true: a cmb_priorityqueue, objects put with the putter's own priority, history
// on (model 13, test/reference/priorityqueue.txt).  The object is the time it was put (a double's bits).
// Oracle: oracle/ref_build/ref_driver.c run_guarded_trial (the counters are described there).
// A template over the engine: GuardedT<cmb::Sim, P, R> is the general-engine model (Guarded<P, R>), and on the static tier
// GuardedT<cmb::StaticSimOf<...>> runs in the tier's second form (static_interrupts) with 7 processes and 2 spare event slots -
// the end event and the nuisance's interrupt, which pops at the time it was made - and a queue window of 32 entries.
#pragma once
#include <type_traits>

#include "../csrc/cmb_kernel.cuh"
#include "../csrc/cmb_static.cuh"

namespace cimba_b200 {
namespace models {

template <class S, bool PRIORITY, bool RECORD>
struct GuardedT {
    typename std::conditional<RECORD, typename S::recorded_queue_type, typename S::queue_type>::type queue;
    typename S::recorded_priorityqueue_type pq;
    uint64_t counter[8];
    double   sum_wait, put_mean, get_mean;
    enum : uint32_t { PUTTER, GETTER, NUISANCE };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER };
    static constexpr uint32_t PUTTERS = 3u, GETTERS = 3u, WORKERS = 6u;
    static constexpr bool static_interrupts = true;
    static constexpr bool static_fel_high = !PRIORITY && !RECORD;     // model 3 reports it (the others their history's size)
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i < PUTTERS ? PUTTER : (i < WORKERS ? GETTER : NUISANCE); }

    CMB_FN void note_signal(int64_t sig, uint32_t which)
    {
        if (sig != CMB_PROCESS_SUCCESS) {
            counter[which] += 1u;
            counter[5] += (uint64_t)sig;
        }
    }

    CMB_FN void putter(S &sim, uint32_t me, int64_t sig)
    {
        GuardedT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(put_mean);
            note_signal(sig, 2u);
            sim.proc[me].u[0] = (uint64_t)__double_as_longlong(cmb_time());
            if (PRIORITY) CMB_PRIORITYQUEUE_PUT(pq, sim.proc[me].u[0], cmb_process_priority(me), nullptr);
            else CMB_OBJECTQUEUE_PUT(queue, sim.proc[me].u[0]);
            if (sig == CMB_PROCESS_SUCCESS) counter[0] += 1u;
            else note_signal(sig, 3u);
        }
        CMB_PROCESS_END
    }

    CMB_FN void getter(S &sim, uint32_t me, int64_t sig)
    {
        GuardedT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(get_mean);
            note_signal(sig, 2u);
            if (PRIORITY) CMB_PRIORITYQUEUE_GET(pq, sim.proc[me].u[0]);
            else CMB_OBJECTQUEUE_GET(queue, sim.proc[me].u[0]);
            if (sig == CMB_PROCESS_SUCCESS) {
                counter[1] += 1u;
                sum_wait = __dadd_rn(sum_wait, __dsub_rn(cmb_time(), __longlong_as_double((long long)sim.proc[me].u[0])));
            }
            else {
                note_signal(sig, 4u);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void nuisance(S &sim, uint32_t me, int64_t sig)
    {
        GuardedT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            {
                const uint32_t victim = (uint32_t)cmb_random_dice(0, (long long)WORKERS - 1);
                const int64_t loud = cmb_random_dice(1, 10);
                const int64_t pri = cmb_random_dice(-5, 5);
                counter[7] += 1u;
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
        if constexpr (PRIORITY) {
            cmb_priorityqueue_initialize(pq, (uint64_t)in.servers);
            cmb_priorityqueue_recording_start(pq);
        }
        else {
            cmb_objectqueue_initialize(queue, (uint64_t)in.servers);
            if constexpr (RECORD) cmb_objectqueue_recording_start(queue);
        }
        for (uint32_t i = 0u; i < WORKERS; i++) {
            const int64_t pri = cmb_random_dice(-5, 5);
            cmb_process_start(cmb_process_create(i < PUTTERS ? PUTTER : GETTER, pri, i));
        }
        cmb_process_start(cmb_process_create(NUISANCE, 0, WORKERS));
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == PUTTER) putter(sim, me, sig);
        else if (kind == GETTER) getter(sim, me, sig);
        else nuisance(sim, me, sig);
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)
    {
        GuardedT &m = *this;
        if (action == END_EVENT) {
            for (uint32_t i = 0u; i <= WORKERS; i++) cmb_process_stop(i, 0);
        }
    }
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        counter[6] = PRIORITY ? cmb_priorityqueue_length(pq) : cmb_objectqueue_length(queue);
        if constexpr (PRIORITY) {
            cmb_priorityqueue_recording_stop(pq);
            counter[6] = (uint64_t)__double_as_longlong(pq.history.acc.m1);
            out.max_queue = (uint32_t)pq.history.acc.count;
        }
        else if constexpr (RECORD) {
            cmb_objectqueue_recording_stop(queue);
            counter[6] = (uint64_t)__double_as_longlong(queue.history.acc.m1);
            out.max_queue = (uint32_t)queue.history.acc.count;
        }
        else {
            out.max_queue = sim.fel_high;
        }
        for (uint32_t i = 0u; i < 8u; i++) out.counters[i] = counter[i];
        out.objects = counter[1];
        out.sum_wait = sum_wait;
    }
};

template <bool PRIORITY, bool RECORD>
using Guarded = GuardedT<cmb::Sim, PRIORITY, RECORD>;

// the three as templates over the engine alone, for the static tier's launch
template <class S> using GuardedQueueT = GuardedT<S, false, false>;             // model 3
template <class S> using GuardedRecordedQueueT = GuardedT<S, false, true>;      // model 11
template <class S> using GuardedPriorityQueueT = GuardedT<S, true, true>;       // model 13

}  // namespace models
}  // namespace cimba_b200
