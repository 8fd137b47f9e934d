// examples/clinic_model.cuh - a walk-in clinic, written from scratch against the authoring surface (cimba_b200/csrc/cmb_device.cuh)
// to draw every cmb_random distribution a model can call, and to keep its statistics in cmb_datasummary / cmb_wtdsummary.
// A template over the engine: the same text runs on the general engine (cmb::Sim, examples/clinic_user_model.cu) and, one
// arrival process, three desks and two queues being all it has, on the static tier (cmb::StaticSim<4, 2>,
// examples/clinic_static_user_model.cu).
//
// Patients arrive in groups: the gaps are hyperexponential (CMB_PROCESS_HOLD_SAMPLED, drawn by the dispatcher), a group is
// geometric(0.6) + binomial(2, 0.25) + negative_binomial(1, 0.8) + pascal(1, 0.9) patients (drawn in that order), and triage sends each group by a Vose alias table (0.5, 0.3, 0.2) to desk 0's queue, to the
// queue that desks 1 and 2 share, or home with advice (counted, not served).  Service times are sampled holds:
//   desk 0: PERT_mod(srv / 4, srv, 3 srv, lambda 4);
//   desk 1: 2 srv std_beta(2, 3) + srv / 10 chisquared(3) + srv / 20 std_gamma(2.5);
//   desk 2: srv / 2 F(5, 10) + Erlang(2, srv / 4) + srv / 10 hypoexponential(srv / 2, srv).
// After each service the desk files the visit under one of four codes by loaded dice.  Values that may be negative (cauchy, t, std_t, logistic) and the
// distributions whose variate is a log or pow (weibull, pareto, gamma with shape < 1), with std_exponential, only go into
// summaries: they never steer the trajectory.
// params[0] picks the summary written to counters[0..7] as a row (cmb_summary_to_counters): 0 = the queue of desk 0 as a
// time-weighted history (cmb_wtdsummary over queue lengths and their durations), 1 = signed values, 2 = log / pow values,
// 3 = group sizes, 4 = visit codes.
// The same clinic written against the reference's API is oracle/ref_build/clinic_driver.c (vectors: tests/golden/clinic_vectors.json).
// Every draw is a statement of its own: C and C++ leave the order of the operands of `+` unspecified.
// objects = patients served; sum_wait = their total time in the clinic; max_queue = patients sent home with advice.
#pragma once
#include "../cimba_b200/csrc/cmb_kernel.cuh"
#include "../cimba_b200/csrc/cmb_static.cuh"

namespace clinic_example {
using namespace cimba_b200;

template <class S>
struct ClinicT {
    typename S::queue_type q0, q1;
    cmb_random_alias<3> route;
    double   arr_mean, srv_mean, hyper_m[3], hyper_p[3], hypo_m[2], codes_p[4];
    uint64_t num_objects, groups, served, advised, group_size, member, stamp, desk;
    double   sum_wait, q0_since;
    uint32_t report;
    cmb_wtdsummary q0_len;
    cmb_datasummary signed_values, logpow_values, sizes, codes;
    enum : uint32_t { ARRIVAL, DESK0, DESK1, DESK2 };
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i; }      // creation order: arrival, then desks 0, 1, 2

    CMB_FN void arrival(S &sim, uint32_t me, int64_t sig)
    {
        ClinicT &m = *this;
        CMB_PROCESS_BEGIN
        for (groups = 0u; groups < num_objects; groups++) {
            CMB_PROCESS_HOLD_SAMPLED(ARRIVAL);
            group_size = cmb_random_geometric(0.6);
            group_size += cmb_random_binomial(2u, 0.25);
            group_size += cmb_random_negative_binomial(1u, 0.8);
            group_size += cmb_random_pascal(1u, 0.9);
            (void)cmb_datasummary_add(&sizes, (double)group_size);
            desk = cmb_random_alias_sample(route);
            if (desk == 2u) {
                advised += group_size;
                continue;
            }
            for (member = 0u; member < group_size; member++) {
                stamp = (uint64_t)__double_as_longlong(cmb_time());
                if (desk == 0u) {
                    q0_sample(sim);
                    CMB_OBJECTQUEUE_PUT(q0, stamp);
                }
                else {
                    CMB_OBJECTQUEUE_PUT(q1, stamp);
                }
            }
        }
        CMB_PROCESS_END
    }

    // desk D (0: queue 0; 1 and 2: queue 1); proc.u[0] = the patient's arrival stamp
    template <uint32_t D>
    CMB_FN void desk_body(S &sim, uint32_t me, int64_t sig)
    {
        ClinicT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            if (D == 0u) {
                q0_sample(sim);
                CMB_OBJECTQUEUE_GET(q0, sim.proc[me].u[0]);
            }
            else {
                CMB_OBJECTQUEUE_GET(q1, sim.proc[me].u[0]);
            }
            CMB_PROCESS_HOLD_SAMPLED(DESK0 + D);
            sum_wait += cmb_time() - __longlong_as_double((long long)sim.proc[me].u[0]);
            served += 1u;
            after_visit(sim);
        }
        CMB_PROCESS_END
    }

    CMB_FN void q0_sample(S &sim)           // desk 0's queue length, sampled at each put and get, weighted by the time it lasted
    {
        (void)cmb_wtdsummary_add(&q0_len, (double)cmb_objectqueue_length(q0), cmb_time() - q0_since);
        q0_since = cmb_time();
    }

    CMB_FN void after_visit(S &sim)
    {
        (void)cmb_datasummary_add(&codes, (double)cmb_random_loaded_dice(4u, codes_p));
        (void)cmb_datasummary_add(&signed_values, cmb_random_cauchy(0.0, 1.0));
        (void)cmb_datasummary_add(&signed_values, cmb_random_std_t_dist(4.0));
        (void)cmb_datasummary_add(&signed_values, cmb_random_t_dist(1.0, 2.0, 5.0));
        (void)cmb_datasummary_add(&signed_values, cmb_random_logistic(0.0, 1.0));
        (void)cmb_datasummary_add(&logpow_values, cmb_random_weibull(1.5, srv_mean));
        (void)cmb_datasummary_add(&logpow_values, cmb_random_pareto(3.0, 1.0));
        (void)cmb_datasummary_add(&logpow_values, cmb_random_gamma(0.5, 1.0));
        (void)cmb_datasummary_add(&logpow_values, cmb_random_std_exponential());
    }

    // the durations of the holds: a pure function of the generator and the parameters
    CMB_FN double sample(S &sim, uint32_t which)
    {
        if (which == ARRIVAL) return cmb_random_hyperexponential(3u, hyper_m, hyper_p);
        if (which == DESK0) return cmb_random_PERT_mod(0.25 * srv_mean, srv_mean, 3.0 * srv_mean, 4.0);
        if (which == DESK1) {
            const double b = cmb_random_std_beta(2.0, 3.0);
            const double c = cmb_random_chisquared(3.0);
            const double g = cmb_random_std_gamma(2.5);
            return 2.0 * srv_mean * b + 0.1 * srv_mean * c + 0.05 * srv_mean * g;
        }
        const double f = cmb_random_F_dist(5.0, 10.0);
        const double e = cmb_random_erlang(2u, 0.25 * srv_mean);
        const double h = cmb_random_hypoexponential(2u, hypo_m);
        return 0.5 * srv_mean * f + e + 0.1 * h;
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        arr_mean = in.arr_mean;
        srv_mean = in.srv_mean;
        num_objects = in.num_objects;
        report = in.num_params > 0u ? (uint32_t)in.params[0] : 0u;
        hyper_m[0] = 0.5 * arr_mean;
        hyper_m[1] = arr_mean;
        hyper_m[2] = 2.5 * arr_mean;
        hyper_p[0] = 0.5;
        hyper_p[1] = 0.3;
        hyper_p[2] = 0.2;
        hypo_m[0] = 0.5 * srv_mean;
        hypo_m[1] = srv_mean;
        codes_p[0] = 0.4;
        codes_p[1] = 0.3;
        codes_p[2] = 0.2;
        codes_p[3] = 0.1;
        const double desks_p[3] = {0.5, 0.3, 0.2};
        cmb_random_alias_create(route, 3u, desks_p);
        served = advised = 0u;
        sum_wait = 0.0;
        q0_since = 0.0;
        cmb_wtdsummary_initialize(&q0_len);
        cmb_datasummary_initialize(&signed_values);
        cmb_datasummary_initialize(&logpow_values);
        cmb_datasummary_initialize(&sizes);
        cmb_datasummary_initialize(&codes);
        cmb_objectqueue_initialize(q0, CMB_UNLIMITED);
        cmb_objectqueue_initialize(q1, CMB_UNLIMITED);
        cmb_process_start(cmb_process_create(ARRIVAL, 0, 0u));
        cmb_process_start(cmb_process_create(DESK0, 0, 0u));
        cmb_process_start(cmb_process_create(DESK1, 0, 0u));
        cmb_process_start(cmb_process_create(DESK2, 0, 0u));
    }
    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == ARRIVAL) arrival(sim, me, sig);
        else if (kind == DESK0) desk_body<0u>(sim, me, sig);
        else if (kind == DESK1) desk_body<1u>(sim, me, sig);
        else desk_body<2u>(sim, me, sig);
    }
    CMB_FN void event(S &, uint32_t, uint32_t, int64_t) {}
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }
    CMB_FN void finish(S &sim, cmb::TrialOut &out)
    {
        q0_sample(sim);
        out.objects = served;
        out.sum_wait = sum_wait;
        out.max_queue = (uint32_t)advised;
        if (report == 1u) cmb_summary_to_counters(out, &signed_values);
        else if (report == 2u) cmb_summary_to_counters(out, &logpow_values);
        else if (report == 3u) cmb_summary_to_counters(out, &sizes);
        else if (report == 4u) cmb_summary_to_counters(out, &codes);
        else cmb_summary_to_counters(out, &q0_len);
    }
};
using Clinic = ClinicT<cmb::Sim>;       // on the general engine; ClinicT<cmb::StaticSim<4, 2>> is the static tier's
}  // namespace clinic_example
