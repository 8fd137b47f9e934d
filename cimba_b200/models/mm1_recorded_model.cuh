// mm1_recorded_model.cuh - the reference's first tutorial (tutorial/tut_1_5.c ... tut_1_7.c) and test/test_cimba.c: the M/M/1 queue
// with the queue's length history switched on, each trial reporting the time-weighted queue length.  benchmark/MM1_multi.c's two
// process bodies plus cmb_objectqueue_recording_start / _stop.  Oracle: oracle/ref_build/ref_driver.c model 9 (the eight words of
// the history's cmb_wtdsummary in counters[0..7]).  A template over the engine like mm1_model.cuh: the general engine, or the
// static tier with a recorded queue (S::recorded_queue_type).
#pragma once
#include "../csrc/cmb_kernel.cuh"
#include "../csrc/cmb_static.cuh"

namespace cimba_b200 {
namespace models {

template <class S>
struct MM1RecordedT {
    typename S::recorded_queue_type queue;
    uint32_t arrival, service;
    double   arr_mean, srv_mean;
    uint64_t num_objects, obj_cnt;
    double   sum_wait;
    uint64_t ui, stamp, object;
    enum : uint32_t { ARRIVAL, SERVICE };
    static constexpr bool exponential_holds_only = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i == 0u ? ARRIVAL : SERVICE; }

    CMB_FN void arrivalfunc(S &sim, uint32_t me, int64_t sig)
    {
        MM1RecordedT &m = *this;
        CMB_PROCESS_BEGIN
        for (ui = 0u; ui < num_objects; ui++) {
            CMB_PROCESS_HOLD_EXPONENTIAL(arr_mean);
            stamp = (uint64_t)__double_as_longlong(cmb_time());
            CMB_OBJECTQUEUE_PUT(queue, stamp);
        }
        CMB_PROCESS_END
    }

    CMB_FN void servicefunc(S &sim, uint32_t me, int64_t sig)
    {
        MM1RecordedT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_OBJECTQUEUE_GET(queue, object);
            CMB_PROCESS_HOLD_EXPONENTIAL(srv_mean);
            sum_wait += cmb_time() - __longlong_as_double((long long)object);
            obj_cnt += 1u;
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        arr_mean = in.arr_mean;
        srv_mean = in.srv_mean;
        num_objects = in.num_objects;
        obj_cnt = 0u;
        sum_wait = 0.0;
        cmb_objectqueue_initialize(queue, CMB_UNLIMITED);
        cmb_objectqueue_recording_start(queue);
        arrival = cmb_process_create(ARRIVAL, 0, 0u);
        cmb_process_start(arrival);
        service = cmb_process_create(SERVICE, 0, 0u);
        cmb_process_start(service);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == ARRIVAL) arrivalfunc(sim, me, sig);
        else servicefunc(sim, me, sig);
    }
    CMB_FN void event(S &, uint32_t, uint32_t, int64_t) {}
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        MM1RecordedT &m = *this;
        cmb_objectqueue_recording_stop(queue);
        cmb_summary_to_counters(out, &queue.history.acc);   // what cmb_timeseries_summarize makes of the stored history
        cmb_process_stop(service, 0);
        out.objects = obj_cnt;
        out.sum_wait = sum_wait;
    }
};

using MM1Recorded = MM1RecordedT<cmb::Sim>;

}  // namespace models
}  // namespace cimba_b200
