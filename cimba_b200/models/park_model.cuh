// park_model.cuh - the reference's third tutorial, tutorial/tut_3_1.c, written against the authoring surface: a theme park of nine
// attractions (M/G/n: 11 priority queues, 14 servers running rides in batches of up to ten), visitors that arrive as a Poisson
// stream for 16 hours, walk from attraction to attraction (a Vose alias table per attraction, PERT walking times), join the
// shortest queue, BALK at a queue longer than their patience allows, JOCKEY to a shorter queue when a first patience timer fires
// (cmb_priorityqueue_position / _cancel / _put with a raised priority), RENEGE when a second one does, and otherwise yield until
// the server that took them (cmb_priorityqueue_get, cmb_process_timers_clear on the VISITOR) has run its ride and resumes them;
// gold-card visitors have process priority 5.  A departure process collects five statistics per visitor.
//
// The park's structure below is the tutorial's hard-coded configuration (tut_3_1.c:56-112, "should be an input file").
// Oracle: the UNMODIFIED tutorial source, seeded and silenced through redirected names (oracle/ref_build/tut3_driver.c ->
// oracle/_ref/libtut3_ref.so); vectors in tests/golden/park_vectors.json.
//   counters[0..4] = mean time in park, riding, waiting, walking, mean number of rides (bits of doubles); [5] = visitors departed;
//   objects = visitors created; sum_wait = sum of the visitors' times in the park.
#pragma once
#include "../csrc/cmb_kernel.cuh"

namespace cimba_b200 {
namespace models {

#ifdef CMB_HOST_BUILD
#define PARK_TABLE static const
#else
#define PARK_TABLE __device__ const
#endif

namespace park {
constexpr uint32_t ATTRACTIONS = 9u, STOPS = 11u, ENTRANCE = 0u, EXIT = 10u;    // entrance, nine attractions, exit
constexpr uint32_t QUEUES = 11u, SERVERS = 14u, MAX_BATCH = 10u;
constexpr double ARRIVAL_RATE = 0.5, GOLDCARDS = 0.25, DURATION = 16 * 60.0;
constexpr unsigned BALKING_THRESHOLD = 10u;
constexpr double JOCKEYING_THRESHOLD = 5.0, RENEGING_THRESHOLD = 10.0;
constexpr int64_t TIMER_JOCKEYING = 17, TIMER_RENEGING = 42;

PARK_TABLE double transition_probs[STOPS][STOPS] = {       // i => j, tut_3_1.c:60-72
    { 0.00, 0.30, 0.20, 0.20, 0.10, 0.05, 0.05, 0.00, 0.00, 0.00, 0.10 },
    { 0.00, 0.00, 0.30, 0.20, 0.10, 0.10, 0.05, 0.05, 0.00, 0.00, 0.20 },
    { 0.00, 0.10, 0.05, 0.20, 0.10, 0.15, 0.05, 0.05, 0.05, 0.05, 0.20 },
    { 0.00, 0.05, 0.10, 0.05, 0.20, 0.10, 0.10, 0.05, 0.05, 0.05, 0.25 },
    { 0.00, 0.05, 0.00, 0.10, 0.05, 0.20, 0.15, 0.10, 0.05, 0.05, 0.25 },
    { 0.00, 0.00, 0.00, 0.05, 0.05, 0.00, 0.20, 0.20, 0.10, 0.10, 0.30 },
    { 0.00, 0.00, 0.00, 0.05, 0.10, 0.05, 0.00, 0.30, 0.10, 0.10, 0.30 },
    { 0.00, 0.00, 0.00, 0.05, 0.05, 0.05, 0.05, 0.05, 0.20, 0.20, 0.35 },
    { 0.00, 0.00, 0.00, 0.00, 0.00, 0.05, 0.05, 0.10, 0.00, 0.30, 0.50 },
    { 0.00, 0.00, 0.00, 0.00, 0.00, 0.00, 0.05, 0.10, 0.20, 0.00, 0.65 },
    { 0.00, 0.00, 0.00, 0.00, 0.00, 0.00, 0.00, 0.00, 0.00, 0.00, 1.00 }
};
PARK_TABLE double transition_times[STOPS][STOPS] = {       // mean walking times, :75-87
    { 0.00, 3.00, 7.00, 8.00, 9.00, 12.0, 13.0, 15.0, 20.0, 25.0, 30.0 },
    { 3.00, 1.00, 3.00, 7.00, 8.00, 9.00, 12.0, 13.0, 15.0, 20.0, 25.0 },
    { 7.00, 3.00, 1.00, 3.00, 7.00, 8.00, 9.00, 12.0, 13.0, 15.0, 20.0 },
    { 8.00, 7.00, 3.00, 1.00, 3.00, 7.00, 8.00, 9.00, 12.0, 13.0, 15.0 },
    { 9.00, 8.00, 7.00, 3.00, 1.00, 3.00, 7.00, 8.00, 9.00, 12.0, 13.0 },
    { 12.0, 9.00, 8.00, 7.00, 3.00, 1.00, 3.00, 7.00, 8.00, 9.00, 12.0 },
    { 13.0, 12.0, 9.00, 8.00, 7.00, 3.00, 1.00, 3.00, 7.00, 8.00, 9.00 },
    { 15.0, 13.0, 12.0, 9.00, 8.00, 7.00, 3.00, 1.00, 3.00, 7.00, 8.00 },
    { 20.0, 15.0, 13.0, 12.0, 9.00, 8.00, 7.00, 3.00, 1.00, 3.00, 7.00 },
    { 25.0, 20.0, 15.0, 13.0, 12.0, 9.00, 8.00, 7.00, 3.00, 1.00, 3.00 },
    { 30.0, 25.0, 20.0, 15.0, 13.0, 12.0, 9.00, 8.00, 7.00, 3.00, 0.00 }
};
PARK_TABLE uint32_t num_queues[STOPS]        = { 0, 1, 1, 1, 3, 1, 1, 1, 1, 1, 0 };     // :90-97
PARK_TABLE uint32_t num_servers_per_q[STOPS] = { 0, 1, 3, 2, 1, 1, 1, 1, 1, 1, 0 };
PARK_TABLE uint32_t batch_sizes[STOPS]       = { 0, 1, 5, 5, 1, 10, 5, 8, 1, 1, 0 };
PARK_TABLE double min_durations[STOPS]  = { 0.0, 3.0, 5.0, 4.0, 15.0,  8.0, 5.0, 5.0, 6.0, 3.0, 0.0 };     // :99-106
PARK_TABLE double mode_durations[STOPS] = { 0.0, 4.0, 6.0, 5.0, 20.0,  9.0, 6.0, 5.5, 7.0, 4.0, 0.0 };
PARK_TABLE double max_durations[STOPS]  = { 0.0, 5.0, 7.0, 6.0, 24.0, 12.0, 8.0, 6.0, 8.0, 5.0, 0.0 };
}  // namespace park

struct Park {
    struct Visitor {                                    // struct visitor, :117-128, plus visitor_proc's locals that outlive a blocking call
        double   patience, entry_time_park, entry_time_queue, riding_time, waiting_time, walking_time, wt;
        uint64_t shrtlen, handle;
        uint32_t current_attraction, num_attractions_visited, ua, nxt, shrtqi, q, next_free, pad;
    };
    cmb::priorityqueue queue[park::QUEUES];
    uint32_t queue_base[park::STOPS];                   // first queue of attraction i
    uint32_t server_queue[park::SERVERS], server_stop[park::SERVERS];
    uint32_t batch[park::SERVERS][park::MAX_BATCH];     // serverfunc's batch[] (:165), one row per server
    cmb_random_alias<park::STOPS> quo_vadis[park::STOPS - 1u];     // each attraction's struct cmb_random_alias (tut_3_1.c's quo_vadis)
    cmb::objectqueue departeds;
    cmb_datasummary time_in_park, riding_times, waiting_times, walking_times, num_rides;
    Visitor  *vis;
    Visitor   vis_inline[8];
    uint32_t  vis_cap, vis_top, vis_free;
    uint32_t  arrivals, departures;
    uint64_t  created, object;
    enum : uint32_t { SERVER, VISITOR, ARRIVAL, DEPARTURE };
    enum : uint32_t { END_SIM = cmb::ACT_CMB_USER };

    // ------------------------------------------------------------------ visitor records (the tutorial mallocs them)
    CMB_FN uint32_t visitor_alloc(cmb::Sim &sim)
    {
        if (vis_free != cmb::NIL) {
            const uint32_t k = vis_free;
            vis_free = vis[k].next_free;
            return k;
        }
        if (vis_top == vis_cap) {
            Visitor *bigger = (Visitor *)sim.arena.alloc((uint64_t)(2u * vis_cap) * sizeof(Visitor));
            if (bigger == nullptr) {
                sim.status |= cmb::TRIAL_ERR_ARENA;
                return 0u;
            }
            for (uint32_t k = 0u; k < vis_top; k++) bigger[k] = vis[k];
            vis = bigger;
            vis_cap *= 2u;
        }
        return vis_top++;
    }

    // shortest of the attraction's queues (visitor_proc :351-362 and again :394-404)
    CMB_FN void shortest_queue(uint32_t stop, uint64_t &len_out, uint32_t &qi_out)
    {
        uint64_t shrtlen = UINT64_MAX;
        uint32_t shrtqi = 0u;
        for (uint32_t qi = 0u; qi < park::num_queues[stop]; qi++) {
            const uint32_t len = (uint32_t)cmb_priorityqueue_length(queue[queue_base[stop] + qi]);
            if (len < shrtlen) {
                shrtlen = len;
                shrtqi = qi;
            }
        }
        len_out = shrtlen;
        qi_out = shrtqi;
    }

    // ------------------------------------------------------------------ serverfunc, :156-199
    // proc.u[0] = cnt, proc.u[1] = the loop index ui, proc.f[0] = dur
    CMB_FN void server(cmb::Sim &sim, uint32_t me, int64_t sig)
    {
        Park &m = *this;
#define PARK_S (sim.proc[me].ctx)
        CMB_PROCESS_BEGIN
        for (;;) {
            sim.proc[me].u[0] = 0u;
            do {
                CMB_PRIORITYQUEUE_GET(queue[server_queue[PARK_S]], object);
                cmb_process_timers_clear((uint32_t)object);
                batch[PARK_S][sim.proc[me].u[0]++] = (uint32_t)object;
            } while (cmb_priorityqueue_length(queue[server_queue[PARK_S]]) > 0u &&
                     sim.proc[me].u[0] < park::batch_sizes[server_stop[PARK_S]]);
            for (sim.proc[me].u[1] = 0u; sim.proc[me].u[1] < sim.proc[me].u[0]; sim.proc[me].u[1]++) {
                Visitor &v = vis[sim.proc[batch[PARK_S][sim.proc[me].u[1]]].ctx];
                v.waiting_time = __dadd_rn(v.waiting_time, __dsub_rn(cmb_time(), v.entry_time_queue));
            }
            sim.proc[me].f[0] = cmb_random_PERT(park::min_durations[server_stop[PARK_S]], park::mode_durations[server_stop[PARK_S]],
                                                park::max_durations[server_stop[PARK_S]]);
            CMB_PROCESS_HOLD(sim.proc[me].f[0]);
            for (sim.proc[me].u[1] = 0u; sim.proc[me].u[1] < sim.proc[me].u[0]; sim.proc[me].u[1]++) {
                const uint32_t pid = batch[PARK_S][sim.proc[me].u[1]];
                Visitor &v = vis[sim.proc[pid].ctx];
                v.riding_time = __dadd_rn(v.riding_time, sim.proc[me].f[0]);
                cmb_process_resume(pid, CMB_PROCESS_SUCCESS);
            }
        }
        CMB_PROCESS_END
#undef PARK_S
    }

    // ------------------------------------------------------------------ visitor_proc, :322-438
    CMB_FN void visitor(cmb::Sim &sim, uint32_t me, int64_t sig)
    {
        Park &m = *this;
#define PARK_V (vis[sim.proc[me].ctx])
        CMB_PROCESS_BEGIN
        PARK_V.current_attraction = park::ENTRANCE;
        while (PARK_V.current_attraction != park::EXIT) {
            PARK_V.ua = PARK_V.current_attraction;
            PARK_V.nxt = cmb_random_alias_sample(quo_vadis[PARK_V.ua]);
            PARK_V.wt = walk_time(sim, park::transition_times[PARK_V.ua][PARK_V.nxt]);
            CMB_PROCESS_HOLD(PARK_V.wt);
            PARK_V.walking_time = __dadd_rn(PARK_V.walking_time, PARK_V.wt);
            PARK_V.current_attraction = PARK_V.nxt;
            if (PARK_V.nxt != park::EXIT) {
                shortest_queue(PARK_V.nxt, PARK_V.shrtlen, PARK_V.shrtqi);
                if (PARK_V.shrtlen > (uint64_t)__dmul_rn(PARK_V.patience, (double)park::BALKING_THRESHOLD)) {
                    continue;                           // balked: on to the next attraction
                }
                cmb_process_timer_set(__dmul_rn(PARK_V.patience, park::JOCKEYING_THRESHOLD), park::TIMER_JOCKEYING);
                (void)cmb_process_timer_add(__dmul_rn(PARK_V.patience, park::RENEGING_THRESHOLD), park::TIMER_RENEGING);
                PARK_V.q = queue_base[PARK_V.nxt] + PARK_V.shrtqi;
                PARK_V.entry_time_queue = cmb_time();
                CMB_PRIORITYQUEUE_PUT(queue[PARK_V.q], me, cmb_process_priority(me), &PARK_V.handle);
                for (;;) {
                    CMB_PROCESS_YIELD();
                    if (sig == park::TIMER_JOCKEYING) {
                        if (jockey(sim, me)) continue;
                    }
                    else if (sig == park::TIMER_RENEGING) {
                        (void)cmb_priorityqueue_cancel(queue[PARK_V.q], PARK_V.handle);
                        cmb_process_timers_clear(me);
                        break;
                    }
                    else {
                        PARK_V.num_attractions_visited++;
                        break;
                    }
                }
            }
        }
        CMB_OBJECTQUEUE_PUT(departeds, me);
        CMB_PROCESS_EXIT(0);
        CMB_PROCESS_END
#undef PARK_V
    }

    CMB_FN double walk_time(cmb::Sim &sim, double mwt)
    {
        return cmb_random_PERT(__dmul_rn(0.5, mwt), mwt, __dmul_rn(2.0, mwt));
    }

    // the jockeying branch, :390-416: true = moved to another queue
    CMB_FN bool jockey(cmb::Sim &sim, uint32_t me)
    {
        Park &m = *this;
        Visitor &v = vis[sim.proc[me].ctx];
        const uint32_t mypos = (uint32_t)cmb_priorityqueue_position(queue[v.q], v.handle);
        shortest_queue(v.nxt, v.shrtlen, v.shrtqi);
        if (v.shrtlen < mypos) {
            (void)cmb_priorityqueue_cancel(queue[v.q], v.handle);
            v.q = queue_base[v.nxt] + v.shrtqi;
            // cmb_priorityqueue_put on an unlimited queue never blocks
            (void)cmb::priorityqueue_try_put(sim, m, queue[v.q], (uint64_t)me, cmb_process_priority(me) + 1, &v.handle);
            return true;
        }
        return false;
    }

    // ------------------------------------------------------------------ arrival_proc, :497-517
    CMB_FN void arrival(cmb::Sim &sim, uint32_t me, int64_t sig)
    {
        Park &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(__ddiv_rn(1.0, park::ARRIVAL_RATE));
            admit(sim);
        }
        CMB_PROCESS_END
    }

    CMB_FN void admit(cmb::Sim &sim)
    {
        const double patience = cmb_random_triangular(0.5, 1.0, 1.5);
        const bool goldcard = cmb_random_bernoulli(park::GOLDCARDS);
        const uint32_t slot = visitor_alloc(sim);
        Visitor &v = vis[slot];
        v.patience = patience;
        v.current_attraction = 0u;
        v.num_attractions_visited = 0u;
        v.riding_time = v.waiting_time = v.walking_time = 0.0;
        created += 1u;
        const uint32_t pid = cmb_process_create(VISITOR, goldcard ? 5 : 0, slot);
        v.entry_time_park = cmb_time();
        cmb_process_start(pid);
    }

    // ------------------------------------------------------------------ departure_proc, :520-548
    CMB_FN void departure(cmb::Sim &sim, uint32_t me, int64_t sig)
    {
        Park &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_OBJECTQUEUE_GET(departeds, object);
            collect(sim, (uint32_t)object);
        }
        CMB_PROCESS_END
    }

    CMB_FN void collect(cmb::Sim &sim, uint32_t pid)
    {
        const uint32_t slot = sim.proc[pid].ctx;
        Visitor &v = vis[slot];
        (void)cmb_datasummary_add(&time_in_park, __dsub_rn(cmb_time(), v.entry_time_park));
        (void)cmb_datasummary_add(&riding_times, v.riding_time);
        (void)cmb_datasummary_add(&waiting_times, v.waiting_time);
        (void)cmb_datasummary_add(&num_rides, (double)v.num_attractions_visited);
        (void)cmb_datasummary_add(&walking_times, v.walking_time);
        v.next_free = vis_free;
        vis_free = slot;
        cmb_process_destroy(pid);
    }

    // ------------------------------------------------------------------ run_trial, :566-620
    CMB_FN void run_trial(cmb::Sim &sim, const cmb::TrialIn &)
    {
        cmb_datasummary_initialize(&time_in_park);
        cmb_datasummary_initialize(&riding_times);
        cmb_datasummary_initialize(&waiting_times);
        cmb_datasummary_initialize(&num_rides);
        cmb_datasummary_initialize(&walking_times);
        vis = vis_inline;
        vis_cap = 8u;
        vis_top = 0u;
        vis_free = cmb::NIL;
        created = 0u;
        uint32_t nq = 0u, ns = 0u;
        for (uint32_t ui = 0u; ui < park::ATTRACTIONS + 1u; ui++) {         // attraction_initialize, :257-289
            queue_base[ui] = nq;
            for (uint32_t qi = 0u; qi < park::num_queues[ui]; qi++) {
                cmb_priorityqueue_initialize(queue[nq], CMB_UNLIMITED);
                cmb_priorityqueue_recording_start(queue[nq]);
                for (uint32_t si = 0u; si < park::num_servers_per_q[ui]; si++) {
                    server_queue[ns] = nq;
                    server_stop[ns] = ui;
                    cmb_process_start(cmb_process_create(SERVER, 0, ns));
                    ns++;
                }
                nq++;
            }
            cmb_random_alias_create(quo_vadis[ui], park::STOPS, park::transition_probs[ui]);
        }
        queue_base[park::EXIT] = nq;
        arrivals = cmb_process_create(ARRIVAL, 0, 0u);
        cmb_process_start(arrivals);
        cmb_objectqueue_initialize(departeds, CMB_UNLIMITED);
        departures = cmb_process_create(DEPARTURE, 0, 0u);
        cmb_process_start(departures);
        (void)cmb_event_schedule(END_SIM, cmb::NIL, 0, park::DURATION, 0);
    }

    CMB_FN void process(cmb::Sim &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == SERVER) server(sim, me, sig);
        else if (kind == VISITOR) visitor(sim, me, sig);
        else if (kind == ARRIVAL) arrival(sim, me, sig);
        else departure(sim, me, sig);
    }

    CMB_FN void event(cmb::Sim &sim, uint32_t action, uint32_t, int64_t)       // end_sim, :551-560
    {
        Park &m = *this;
        if (action == END_SIM) cmb_process_stop(arrivals, 0);
    }
    CMB_FN bool demand(cmb::Sim &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(cmb::Sim &, cmb::TrialOut &out)                          // :623-637: the five cmb_datasummary_mean
    {
        out.counters[0] = (uint64_t)__double_as_longlong(cmb_datasummary_mean(&time_in_park));
        out.counters[1] = (uint64_t)__double_as_longlong(cmb_datasummary_mean(&riding_times));
        out.counters[2] = (uint64_t)__double_as_longlong(cmb_datasummary_mean(&waiting_times));
        out.counters[3] = (uint64_t)__double_as_longlong(cmb_datasummary_mean(&walking_times));
        out.counters[4] = (uint64_t)__double_as_longlong(cmb_datasummary_mean(&num_rides));
        out.counters[5] = cmb_datasummary_count(&time_in_park);
        out.objects = created;
        out.sum_wait = __dmul_rn(cmb_datasummary_mean(&time_in_park), (double)cmb_datasummary_count(&time_in_park));
    }

    static uint64_t arena_bytes_per_trial(const cimba_b200_device_job &) { return 131072u; }
};

}  // namespace models
}  // namespace cimba_b200
