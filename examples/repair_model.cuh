// examples/repair_model.cuh - a machine shop, written from scratch against the authoring surface
// (cimba_b200/csrc/cmb_device.cuh): M machines break down, wait for a repair crew shared by all of them (a cmb_resourcepool of
// `servers` units, its usage history on), are repaired, then pass one shared inspection bench (a cmb_resource).
// examples/repair_user_model.cu exports it on the general engine; the same model written against the reference's API is
// oracle/ref_build/repair_driver.c.  With at most eight machines, priority 0 and nothing that interrupts, it also
// runs on the static tier (cmb::StaticSim<8, 0>, examples/repair_static_user_model.cu).
//
// Machine i repeats num_objects times: up time (exponential, arr_mean); acquire `need` crew (1 + (i & 1) with two or more
// crew, else 1 - so with a busy crew a claim is often met in two grabs); repair (exponential, srv_mean); release the crew;
// inspection at the bench (exponential, srv_mean / 4); its downtime added up.
// params[0] = machines (default 8; more than eight: the trial goes to the general engine), params[1] != 0: each machine's
// last cycle ends with CMB_PROCESS_EXIT right after its repair, still holding its crew (the exit drops it).
// Results: objects = repairs, sum_wait = total downtime, counters[0] = acquisitions that found 0 < available < need,
// counters[1] = bench acquisitions that found it held, counters[2..6] = the crew history's count, m1, m2, wsum and max.
#pragma once
#include "../cimba_b200/csrc/cmb_kernel.cuh"
#include "../cimba_b200/csrc/cmb_static.cuh"

namespace repair_example {
using namespace cimba_b200;

template <class S>
struct RepairT {
    typename S::recorded_resourcepool_type crew;
    typename S::resource_type bench;
    double   arr_mean, srv_mean;
    uint64_t num_objects, repairs, partial_grabs, bench_busy;
    double   downtime;
    int32_t  servers;
    bool     exit_holding;
    enum : uint32_t { MACHINE };
    static CMB_FN constexpr uint32_t static_kind(uint32_t) { return MACHINE; }
    static constexpr bool exponential_holds_only = true;    // every draw is a CMB_PROCESS_HOLD_EXPONENTIAL

    CMB_FN uint64_t need(uint32_t i) const { return servers >= 2 ? 1u + (i & 1u) : 1u; }

    // u[0] = cycles done, f[0] = when the machine failed
    CMB_FN void machine(S &sim, uint32_t me, int64_t sig)
    {
        RepairT &m = *this;
        CMB_PROCESS_BEGIN
        for (sim.proc[me].u[0] = 0u; sim.proc[me].u[0] < num_objects; sim.proc[me].u[0]++) {
            CMB_PROCESS_HOLD_EXPONENTIAL(arr_mean);
            sim.proc[me].f[0] = cmb_time();
            if (cmb_resourcepool_available(crew) > 0u && cmb_resourcepool_available(crew) < need(me)) partial_grabs += 1u;
            CMB_RESOURCEPOOL_ACQUIRE(crew, need(me));
            CMB_PROCESS_HOLD_EXPONENTIAL(srv_mean);
            if (exit_holding && sim.proc[me].u[0] + 1u == num_objects) CMB_PROCESS_EXIT(0);
            CMB_RESOURCEPOOL_RELEASE(crew, need(me));
            if (bench.holder != cmb::NIL) bench_busy += 1u;
            CMB_RESOURCE_ACQUIRE(bench);
            CMB_PROCESS_HOLD_EXPONENTIAL(0.25 * srv_mean);
            CMB_RESOURCE_RELEASE(bench);
            downtime += cmb_time() - sim.proc[me].f[0];
            repairs += 1u;
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        arr_mean = in.arr_mean;
        srv_mean = in.srv_mean;
        num_objects = in.num_objects;
        servers = in.servers;
        exit_holding = in.num_params > 1u && in.params[1] != 0.0;
        const uint32_t machines = in.num_params > 0u && in.params[0] > 0.0 ? (uint32_t)in.params[0] : 8u;
        repairs = partial_grabs = bench_busy = 0u;
        downtime = 0.0;
        cmb_resourcepool_initialize(crew, (uint64_t)in.servers);
        cmb_resourcepool_start_recording(crew);
        cmb_resource_initialize(bench);
        for (uint32_t i = 0u; i < machines; i++) cmb_process_start(cmb_process_create(MACHINE, 0, i));
    }
    CMB_FN void process(S &sim, uint32_t me, uint32_t, int64_t sig) { machine(sim, me, sig); }
    CMB_FN void event(S &, uint32_t, uint32_t, int64_t) {}
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }
    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        cmb_resourcepool_stop_recording(crew);
        const WtdAcc &h = crew.history.acc;             // what cmb_timeseries_summarize makes of the stored history
        out.objects = repairs;
        out.sum_wait = downtime;
        out.counters[0] = partial_grabs;
        out.counters[1] = bench_busy;
        out.counters[2] = h.count;
        out.counters[3] = (uint64_t)__double_as_longlong(h.m1);
        out.counters[4] = (uint64_t)__double_as_longlong(h.m2);
        out.counters[5] = (uint64_t)__double_as_longlong(h.wsum);
        out.counters[6] = (uint64_t)__double_as_longlong(h.max);
        out.counters[7] = 0u;
    }
};
using Repair = RepairT<cmb::Sim>;     // on the general engine; RepairT<cmb::StaticSim<8, 0>> is the static tier's
}  // namespace repair_example
