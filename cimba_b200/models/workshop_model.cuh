// workshop_model.cuh - the reference's buffer and resource tests written against the authoring surface.
//
// WorkshopT<S, PLAIN> (Workshop<PLAIN> on the general engine): test/test_buffer.c and test/test_resource.c in one world - fillers
// and drainers moving random amounts
// through a cmb_buffer of capacity `servers`, a polite and a pre-empting worker sharing one cmb_resource, a nuisance
// interrupting all six, an end event stopping everybody.  PLAIN = false: two fillers, two drainers, two workers, amounts
// 1..8 (model 5); PLAIN = true: test/test_buffer.c as it stands - three fillers, three drainers, amounts 1..15, the level
// history on (model 12, golden file test/reference/buffer.txt).  A template over the engine: cmb::Sim, or the static tier's second
// form, where the buffer's guards are literal heaps.
// Tool: test/test_resource.c as it stands - three targets with random priorities and a pre-empter (priority 0) on one
// cmb_resource with its history on (model 14, golden file test/reference/resource.txt).  A template over the engine, as
// tutorial1_model.cuh: cmb::Sim, or the static tier's second form (static_interrupts: priorities, pre-emption).
// Oracle: oracle/ref_build/ref_driver.c run_buffer_trial / run_resource_trial (the counters are described there).
#pragma once
#include "../csrc/cmb_kernel.cuh"
#include "../csrc/cmb_static.cuh"

namespace cimba_b200 {
namespace models {

// A template over the engine: WorkshopT<cmb::Sim, PLAIN> is the general-engine model (Workshop<PLAIN>); on the static tier both
// forms run in the second form with 7 processes and WORKSHOP_SPARE_SLOTS spare event slots for the end event, the nuisance's
// interrupt and the pre-empting worker's ACT_CMB_WAKE_PREEMPT.  2 is the fewest at which no vector case of
// tests/golden/cmb_engine_vectors.json flags (with 1, all do); a trial that needs more is flagged and re-run on the general engine.
constexpr int WORKSHOP_SPARE_SLOTS = 2;

template <class S, bool PLAIN>
struct WorkshopT {
    typename std::conditional<PLAIN, typename S::recorded_buffer_type, typename S::buffer_type>::type store;
    typename S::resource_type tool;
    uint64_t counter[8];
    double   sum_wait, put_mean, get_mean;
    enum : uint32_t { FILLER, DRAINER, WORKER, NUISANCE };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER };
    static constexpr uint32_t PROCS = 6u;
    static constexpr long long AMOUNT_MAX = PLAIN ? 15 : 8;
    static constexpr uint32_t FILLERS = PLAIN ? 3u : 2u, DRAINERS = PLAIN ? 3u : 2u;
    static constexpr bool static_interrupts = true;
    static constexpr bool static_fel_high = !PLAIN;
    static constexpr int static_min_ctas = 1;       // without it ptxas holds the kernels to 96 registers and spills
    static CMB_FN constexpr uint32_t static_kind(uint32_t i)
    {
        return i < FILLERS ? FILLER : i < FILLERS + DRAINERS ? DRAINER : i < PROCS ? WORKER : NUISANCE;
    }
    template <class F>
    CMB_FN void static_holdables(F &&visit) { visit(tool); }

    CMB_FN void note(int64_t sig)
    {
        if (sig != CMB_PROCESS_SUCCESS) counter[6] += (uint64_t)sig;
    }

    // u[0] = the amount offered / wanted, u[1] = what the call left of it
    CMB_FN void filler(S &sim, uint32_t me, int64_t sig)
    {
        WorkshopT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(put_mean);
            note(sig);
            sim.proc[me].u[0] = (uint64_t)cmb_random_dice(1, AMOUNT_MAX);
            sim.proc[me].u[1] = sim.proc[me].u[0];
            CMB_BUFFER_PUT(store, sim.proc[me].u[1]);
            counter[0] += sim.proc[me].u[0] - sim.proc[me].u[1];
            if (sig != CMB_PROCESS_SUCCESS) {
                counter[2] += 1u;
                note(sig);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void drainer(S &sim, uint32_t me, int64_t sig)
    {
        WorkshopT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(get_mean);
            note(sig);
            sim.proc[me].u[1] = (uint64_t)cmb_random_dice(1, AMOUNT_MAX);
            CMB_BUFFER_GET(store, sim.proc[me].u[1]);
            counter[1] += sim.proc[me].u[1];
            if (sig != CMB_PROCESS_SUCCESS) {
                counter[3] += 1u;
                note(sig);
            }
        }
        CMB_PROCESS_END
    }

    // f[0] = when the tool was taken
    CMB_FN void worker(S &sim, uint32_t me, int64_t sig)
    {
        WorkshopT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            if (me == 5u) CMB_RESOURCE_PREEMPT(tool);
            else CMB_RESOURCE_ACQUIRE(tool);
            if (sig == CMB_PROCESS_SUCCESS) {
                counter[4] += 1u;
                sim.proc[me].f[0] = cmb_time();
                CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
                if (sig == CMB_PROCESS_PREEMPTED) {
                    counter[5] += 1u;
                    note(sig);
                }
                else {
                    note(sig);
                    CMB_RESOURCE_RELEASE(tool);
                    sum_wait = __dadd_rn(sum_wait, __dsub_rn(cmb_time(), sim.proc[me].f[0]));
                }
            }
            else {
                note(sig);
            }
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            note(sig);
        }
        CMB_PROCESS_END
    }

    CMB_FN void nuisance(S &sim, uint32_t me, int64_t sig)
    {
        WorkshopT &m = *this;
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
        cmb_buffer_initialize(store, (uint64_t)in.servers);
        if constexpr (PLAIN) cmb_buffer_recording_start(store);
        cmb_resource_initialize(tool);
        const uint32_t fillers = PLAIN ? 3u : 2u, drainers = PLAIN ? 3u : 2u;
        for (uint32_t i = 0u; i < PROCS; i++) {
            const int64_t pri = cmb_random_dice(-5, 5);
            cmb_process_start(cmb_process_create(i < fillers ? FILLER : (i < fillers + drainers ? DRAINER : WORKER), pri, i));
        }
        cmb_process_start(cmb_process_create(NUISANCE, 0, PROCS));
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == FILLER) filler(sim, me, sig);
        else if (kind == DRAINER) drainer(sim, me, sig);
        else if (kind == WORKER) worker(sim, me, sig);
        else nuisance(sim, me, sig);
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)
    {
        WorkshopT &m = *this;
        if (action == END_EVENT) {
            for (uint32_t i = 0u; i <= PROCS; i++) cmb_process_stop(i, 0);
        }
    }
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        counter[7] = cmb_buffer_level(store);
        if constexpr (PLAIN) {
            cmb_buffer_recording_stop(store);
            counter[4] = (uint64_t)__double_as_longlong(store.history.acc.m1);
            out.max_queue = (uint32_t)store.history.acc.count;
        }
        else {
            out.max_queue = sim.fel_high;
        }
        for (uint32_t i = 0u; i < 8u; i++) out.counters[i] = counter[i];
        out.objects = counter[1];
        out.sum_wait = sum_wait;
    }
};

template <bool PLAIN>
using Workshop = WorkshopT<cmb::Sim, PLAIN>;

// the two as templates over the engine alone, for the static tier's launch
template <class S> using WorkshopBufferT = WorkshopT<S, false>;        // model 5
template <class S> using WorkshopRecordedT = WorkshopT<S, true>;       // model 12

template <class S>
struct ToolT {
    typename S::recorded_resource_type res;
    uint64_t counter[8];
    double   sum_wait;
    enum : uint32_t { TARGET, PREEMPTER };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER };
    static constexpr bool static_interrupts = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i < 3u ? TARGET : PREEMPTER; }
    template <class F>
    CMB_FN void static_holdables(F &&visit) { visit(res); }

    CMB_FN void target(S &sim, uint32_t me, int64_t sig)
    {
        ToolT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_RESOURCE_ACQUIRE(res);
            if (sig == CMB_PROCESS_SUCCESS) {
                counter[0] += 1u;
                sim.proc[me].f[0] = cmb_time();
                CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
                if (sig == CMB_PROCESS_SUCCESS) {
                    CMB_RESOURCE_RELEASE(res);
                    sum_wait = __dadd_rn(sum_wait, __dsub_rn(cmb_time(), sim.proc[me].f[0]));
                }
                else {
                    counter[1] += 1u;
                    if (counter[5] == 0u) {
                        counter[4] = (uint64_t)__double_as_longlong(cmb_time());
                        counter[5] = (uint64_t)me + 1u;
                    }
                }
            }
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
        }
        CMB_PROCESS_END
    }

    CMB_FN void preempter(S &sim, uint32_t me, int64_t sig)
    {
        ToolT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_RESOURCE_PREEMPT(res);
            counter[2] += 1u;
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
            CMB_RESOURCE_RELEASE(res);
            CMB_PROCESS_HOLD_EXPONENTIAL(1.0);
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        for (uint32_t i = 0u; i < 8u; i++) counter[i] = 0u;
        sum_wait = 0.0;
        cmb_resource_initialize(res);
        cmb_resource_start_recording(res);
        for (uint32_t i = 0u; i < 3u; i++) {
            const int64_t pri = cmb_random_dice(-5, 5);
            cmb_process_start(cmb_process_create(TARGET, pri, i));
        }
        cmb_process_start(cmb_process_create(PREEMPTER, 0, 3u));
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == TARGET) target(sim, me, sig);
        else preempter(sim, me, sig);
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)
    {
        ToolT &m = *this;
        if (action == END_EVENT) {
            for (uint32_t i = 0u; i < 4u; i++) cmb_process_stop(i, 0);
        }
    }
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        cmb_resource_stop_recording(res);
        counter[3] = (uint64_t)__double_as_longlong(res.history.acc.m1);
        for (uint32_t i = 0u; i < 8u; i++) out.counters[i] = counter[i];
        out.max_queue = (uint32_t)res.history.acc.count;
        out.objects = counter[0] + counter[2];
        out.sum_wait = sum_wait;
    }
};

using Tool = ToolT<cmb::Sim>;     // on the static tier: ToolT<cmb::StaticSimOf<ToolT, 4, 0, 2>> (four processes, two spare event slots)

}  // namespace models
}  // namespace cimba_b200
