// harbor_general_model.cuh - the reference's harbor (test/test_condition.c:60-520 = tutorial/tut_4_1.c) written against the
// authoring surface: a weather and a tide process that update the state every hour and signal the harbormaster
// (cmb_condition_signal: every waiter whose predicate holds), an arrival process that creates one ship PROCESS per arrival,
// ships that wait on the harbormaster until depth, wind, tugs and a berth all suit them (cmb_condition_wait with a
// predicate, spurious wake-ups re-tested), take a berth and tugs from three cmb_resourcepools, dock, unload, undock, join the
// departed list and signal Davy Jones, whose departure process collects their exit values and frees them; a process that
// ticks once a year; an end event that stops everybody, ships still active in arrival order.
// The fused kernels (harbor_model.cuh) are what runs this model fast; this is the same model on the general engine
// (job->variant = CIMBA_B200_VARIANT_GENERAL) - the tutorial as a model author would write it - held to the same oracle
// (oracle/ref_build/ref_driver.c model 10) and, like them, to the reference's golden file test/reference/condition.txt.
#pragma once
#include "../csrc/cmb_kernel.cuh"

namespace cimba_b200 {
namespace models {

struct HarborGeneral {
    double   wind_magnitude, wind_direction, water_depth;      // struct env_state, test_condition.c:61-65
    cmb::resourcepool tugs, berths[2];
    cmb::condition harbormaster, davyjones;
    cmb::HashHeap<cmb::EventOrder> active;                      // sim->active_ships: key = ship id, rank = arrival time
    cmb::Tag active_store[9];
    uint32_t departed;                                          // LIFO of departed ships (through Process::u[1]), NIL = empty
    uint32_t weather, tide, arrivals, departures, dots;
    cmb_datasummary through[2];                                      // trl->system_time[size]
    double   arr_mean, unload_small, sum_system_time;
    uint64_t cnt, alive, most_alive, reactivated, left[2];
    enum : uint32_t { WEATHER, TIDE, ARRIVALS, SHIP, DEPARTURES, DOTS };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER };
    enum : uint32_t { CAN_DOCK = cmb::DEMAND_USER, SOMEBODY_LEFT };

    // a ship: ctx = size (0 small, 1 large), u[0] = id, u[1] = next departed, f[0] = arrival time, f[1] = time in system
    static CMB_FN uint32_t tugs_of(uint32_t size) { return size == 0u ? 1u : 3u; }
    CMB_FN double unloading_mean(cmb::Sim &sim, uint32_t pid) { return sim.proc[pid].ctx == 0u ? unload_small : 1.5 * unload_small; }

    static uint64_t arena_bytes_per_trial(const cimba_b200_device_job &) { return 96u * 1024u; }

    CMB_FN bool can_dock(cmb::Sim &sim, uint32_t pid)           // is_ready_to_dock, :189-231
    {
        const uint32_t size = sim.proc[pid].ctx;
        if (water_depth < (size == 0u ? 8.0 : 13.0)) return false;
        if (wind_magnitude > (size == 0u ? 10.0 : 12.0)) return false;
        if (cmb_resourcepool_available(tugs) < tugs_of(size)) return false;
        return cmb_resourcepool_available(berths[size]) >= 1u;
    }

    CMB_FN void weather_proc(cmb::Sim &sim, uint32_t me, int64_t sig)       // :103-137
    {
        HarborGeneral &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            {
                const double gust = cmb_random_rayleigh(5.0);
                wind_magnitude = 0.5 * gust + 0.5 * wind_magnitude;
                const double d1 = cmb_random_PERT(0.0, 225.0, 360.0);
                const double d2 = cmb_random_PERT(0.0, 45.0, 360.0);
                wind_direction = 0.75 * d1 + 0.25 * d2;
                reactivated += cmb_condition_signal(harbormaster);
            }
            CMB_PROCESS_HOLD(1.0);
        }
        CMB_PROCESS_END
    }

    CMB_FN void tide_proc(cmb::Sim &sim, uint32_t me, int64_t sig)          // :140-186
    {
        HarborGeneral &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            {
                const double PI = 3.14159265358979323846;
                const double half_month = 0.5 * 29.5 * 24.0;
                const double t = fmod(cmb_time(), half_month);
                const double astro = 15.0 + 1.0 * sin(2.0 * PI * t / 12.4) + 0.5 * sin(2.0 * PI * t / 24.0)
                                   + 0.25 * sin(2.0 * PI * t / (0.5 * 29.5 * 24));
                const double surge = 0.5 * wind_magnitude - 0.5 * wind_magnitude * sin(wind_direction * PI / 180.0);
                water_depth = astro + surge;
                reactivated += cmb_condition_signal(harbormaster);
            }
            CMB_PROCESS_HOLD(1.0);
        }
        CMB_PROCESS_END
    }

    CMB_FN void ship_proc(cmb::Sim &sim, uint32_t me, int64_t sig)          // :234-320
    {
        HarborGeneral &m = *this;
        CMB_PROCESS_BEGIN
        sim.proc[me].f[0] = cmb_time();
        if (active.enqueue(sim.arena, sim.proc[me].u[0], cmb_time(), 0, me, 0u, 0, cmb::NIL) == 0u) sim.status |= cmb::TRIAL_ERR_ARENA;
        if (++alive > most_alive) most_alive = alive;
        while (!can_dock(sim, me)) {                    // spurious wake-ups: somebody else may have taken the tugs
            CMB_CONDITION_WAIT(harbormaster, CAN_DOCK, 0);
        }
        CMB_RESOURCEPOOL_ACQUIRE(berths[sim.proc[me].ctx], 1u);
        CMB_RESOURCEPOOL_ACQUIRE(tugs, tugs_of(sim.proc[me].ctx));
        CMB_PROCESS_HOLD(cmb_random_PERT(0.4, 0.5, 0.8));
        CMB_RESOURCEPOOL_RELEASE(tugs, tugs_of(sim.proc[me].ctx));
        // (no initialised local may be in scope at a blocking call - the body is re-entered past it: the mean goes through a helper)
        CMB_PROCESS_HOLD(cmb_random_PERT(0.75 * unloading_mean(sim, me), unloading_mean(sim, me), 2 * unloading_mean(sim, me)));
        CMB_RESOURCEPOOL_ACQUIRE(tugs, tugs_of(sim.proc[me].ctx));
        CMB_PROCESS_HOLD(cmb_random_PERT(0.4, 0.5, 0.8));
        CMB_RESOURCEPOOL_RELEASE(berths[sim.proc[me].ctx], 1u);
        CMB_RESOURCEPOOL_RELEASE(tugs, tugs_of(sim.proc[me].ctx));
        (void)active.remove(sim.arena, sim.proc[me].u[0]);
        alive--;
        sim.proc[me].u[1] = departed;                   // cmi_slist_push(sim->departed_ships, ...)
        departed = me;
        (void)cmb_condition_signal(davyjones);
        sim.proc[me].f[1] = cmb_time() - sim.proc[me].f[0];
        CMB_PROCESS_END                                 // returning = cmb_process_exit(the time in system)
    }

    CMB_FN void arrival_proc(cmb::Sim &sim, uint32_t me, int64_t sig)       // :323-377
    {
        HarborGeneral &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(arr_mean);
            {
                const uint32_t size = cmb_random_bernoulli(0.25);
                const uint32_t ship = cmb_process_create(SHIP, 0, size);
                sim.proc[ship].u[0] = ++cnt;
                cmb_process_start(ship);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void departure_proc(cmb::Sim &sim, uint32_t me, int64_t sig)     // :396-432
    {
        HarborGeneral &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_CONDITION_WAIT(davyjones, SOMEBODY_LEFT, 0);    // the only waiter: no loop (:406)
            {
                const uint32_t ship = departed;
                departed = (uint32_t)sim.proc[ship].u[1];
                const double t_sys = sim.proc[ship].f[1];       // cmb_process_exit_value
                const uint32_t size = sim.proc[ship].ctx;
                (void)cmb_datasummary_add(&through[size], t_sys);
                sum_system_time += t_sys;
                left[size] += 1u;
                cmb_process_destroy(ship);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void dots_proc(cmb::Sim &sim, uint32_t me, int64_t sig)          // :435-448
    {
        HarborGeneral &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD(24.0 * 7 * 52);
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(cmb::Sim &sim, const cmb::TrialIn &in)           // test_condition, :490-560 (creation order as the oracle's)
    {
        HarborGeneral &m = *this;
        (void)&m;
        wind_magnitude = wind_direction = water_depth = 0.0;
        arr_mean = in.arr_mean;
        unload_small = in.srv_mean;
        sum_system_time = 0.0;
        cnt = alive = most_alive = reactivated = 0u;
        left[0] = left[1] = 0u;
        cmb_datasummary_initialize(&through[0]);
        cmb_datasummary_initialize(&through[1]);
        departed = cmb::NIL;
        weather = cmb_process_create(WEATHER, 0, 0u);
        cmb_process_start(weather);
        tide = cmb_process_create(TIDE, 0, 0u);
        cmb_process_start(tide);
        cmb_resourcepool_initialize(tugs, (uint64_t)in.servers);
        cmb_resourcepool_start_recording(tugs);
        cmb_resourcepool_initialize(berths[0], 6u);
        cmb_resourcepool_start_recording(berths[0]);
        cmb_resourcepool_initialize(berths[1], 3u);
        cmb_resourcepool_start_recording(berths[1]);
        cmb_condition_initialize(harbormaster);
        cmb_condition_initialize(davyjones);
        arrivals = cmb_process_create(ARRIVALS, 0, 0u);
        cmb_process_start(arrivals);
        departures = cmb_process_create(DEPARTURES, 0, 0u);
        cmb_process_start(departures);
        active.init(active_store, 3u);
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
        dots = cmb_process_create(DOTS, 0, 0u);
        cmb_process_start(dots);
    }

    CMB_FN void process(cmb::Sim &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        switch (kind) {
        case WEATHER:    weather_proc(sim, me, sig); break;
        case TIDE:       tide_proc(sim, me, sig); break;
        case ARRIVALS:   arrival_proc(sim, me, sig); break;
        case SHIP:       ship_proc(sim, me, sig); break;
        case DEPARTURES: departure_proc(sim, me, sig); break;
        default:         dots_proc(sim, me, sig); break;
        }
    }

    CMB_FN void event(cmb::Sim &sim, uint32_t action, uint32_t, int64_t)   // end_sim_evt, :451-474
    {
        HarborGeneral &m = *this;
        if (action != END_EVENT) return;
        cmb_process_stop(weather, 0);
        cmb_process_stop(tide, 0);
        cmb_process_stop(arrivals, 0);
        cmb_process_stop(departures, 0);
        cmb_process_stop(dots, 0);
        while (active.count > 0u) {                     // ships still active, in arrival order
            (void)active.dequeue();
            const uint32_t ship = active.tag[0].subj;
            cmb_process_stop(ship, 0);
            cmb_process_destroy(ship);
        }
    }

    CMB_FN bool demand(cmb::Sim &sim, uint32_t id, uint32_t pid, int32_t)
    {
        return id == CAN_DOCK ? can_dock(sim, pid) : departed != cmb::NIL;  // is_ready_to_dock / is_departed (:380-393)
    }

    CMB_FN void finish(cmb::Sim &, cmb::TrialOut &out)
    {
        out.counters[0] = left[0];
        out.counters[1] = left[1];
        out.counters[2] = (uint64_t)__double_as_longlong(cmb_datasummary_mean(&through[0]));
        out.counters[3] = (uint64_t)__double_as_longlong(cmb_datasummary_mean(&through[1]));
        out.counters[4] = tugs.history.acc.count;       // history samples with a duration (recording is never stopped)
        out.counters[5] = (uint64_t)__double_as_longlong(tugs.history.acc.m1);
        out.counters[6] = berths[0].history.acc.count | (berths[1].history.acc.count << 32);
        out.counters[7] = reactivated;
        out.objects = left[0] + left[1];
        out.sum_wait = sum_system_time;
        out.max_queue = (uint32_t)most_alive;
    }
};

}  // namespace models
}  // namespace cimba_b200
