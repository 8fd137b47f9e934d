// tutorial1_model.cuh - the trial of the reference's first tutorial, tutorial/tut_1_7.c (run_MM1_trial :155-222, the processes
// :107-151, the events :69-101), written against the authoring surface: an M/M/1 queue held in a cmb_buffer (amounts of 1), an
// event that switches the level history on at the warm-up time, one that switches it off at warm-up + duration, and an end event
// of priority -100 at the same time that stops both processes.  What the tutorial reports per trial is the time-weighted mean
// level (its avg_queue_length); here the whole cmb_wtdsummary goes to counters[0..7].
//   arr_mean / srv_mean = 1 / arr_rate, 1 / srv_rate; num_objects = duration; params[0] = warm-up time.
// Oracle: oracle/ref_build/ref_driver.c model 19 (the same trial against the reference's API).
// A template over the engine: cmb::Sim (general), or cmb::StaticSim<2, 0, 3> - the static tier with a cmb_buffer, three slots for
// the model's own events and the event list ordered by priority as well.
#pragma once
#include "../csrc/cmb_kernel.cuh"
#include "../csrc/cmb_static.cuh"

namespace cimba_b200 {
namespace models {

template <class S>
struct Tutorial1T {
    typename S::recorded_buffer_type que;                                    // struct simulation, tut_1_7.c:36-41
    uint32_t arr, srv;
    double   t_ia_mean, t_srv_mean;                     // 1 / arr_rate, 1 / srv_rate (:117, :141)
    uint64_t n, units_put, units_got;
    enum : uint32_t { ARRIVAL, SERVICE };
    enum : uint32_t { START_REC = cmb::ACT_CMB_USER, STOP_REC, END_SIM };
    static constexpr bool exponential_holds_only = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i == 0u ? ARRIVAL : SERVICE; }

    CMB_FN void arrival(S &sim, uint32_t me, int64_t sig)               // :107-128
    {
        Tutorial1T &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(t_ia_mean);
            n = 1u;
            CMB_BUFFER_PUT(que, n);
            units_put += 1u;
        }
        CMB_PROCESS_END
    }

    CMB_FN void service(S &sim, uint32_t me, int64_t sig)               // :133-151
    {
        Tutorial1T &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            n = 1u;
            CMB_BUFFER_GET(que, n);
            units_got += 1u;
            CMB_PROCESS_HOLD_EXPONENTIAL(t_srv_mean);
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)               // :155-200
    {
        t_ia_mean = in.arr_mean;
        t_srv_mean = in.srv_mean;
        units_put = units_got = 0u;
        cmb_buffer_initialize(que, CMB_UNLIMITED);
        arr = cmb_process_create(ARRIVAL, 0, 0u);
        cmb_process_start(arr);
        srv = cmb_process_create(SERVICE, 0, 0u);
        cmb_process_start(srv);
        double t = in.num_params > 0u ? in.params[0] : 0.0;                     // warmup_time
        (void)cmb_event_schedule(START_REC, cmb::NIL, 0, t, 0);
        t = __dadd_rn(t, (double)in.num_objects);                               // t += trl->duration
        (void)cmb_event_schedule(STOP_REC, cmb::NIL, 0, t, 0);
        (void)cmb_event_schedule(END_SIM, cmb::NIL, 0, t, -100);               // after everything else at that time
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == ARRIVAL) arrival(sim, me, sig);
        else service(sim, me, sig);
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)       // start_rec, stop_rec, end_sim, :69-101
    {
        Tutorial1T &m = *this;
        if (action == START_REC) {
            cmb_buffer_recording_start(que);
        }
        else if (action == STOP_REC) {
            cmb_buffer_recording_stop(que);
        }
        else if (action == END_SIM) {
            cmb_process_stop(arr, 0);
            cmb_process_stop(srv, 0);
        }
    }
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &, cmb::TrialOut &out)                          // :205-209: cmb_timeseries_summarize of the history
    {
        cmb_summary_to_counters(out, &que.history.acc);                         // counters[3] = avg_queue_length
        out.objects = units_put;
        out.sum_wait = (double)units_got;
    }
};

using Tutorial1 = Tutorial1T<cmb::Sim>;      // on the static tier: Tutorial1T<cmb::StaticSim<2, 0, 3>> (two processes, no object queue, three events)

}  // namespace models
}  // namespace cimba_b200
