// tests/random_sweep_model.cuh - TEST INFRASTRUCTURE: the cmb_random parameter sweep (tests/random_sweep_cases.py) as model code, one
// trial per case.  The case table is compiled in from random_sweep_table.h, which the tests write from the Python table
// (random_sweep_cases.write_model_table) and put on the include path; trial `in.trial` runs case `in.trial`.
//
// One process draws the case's NDRAW variates with the cmb_random_* names of model code.  Where the case's `held` flag is set
// (every variate a finite duration >= 0, proven on the host build first), it then draws NDRAW more as the durations of
// CMB_PROCESS_HOLD_SAMPLED: sample() stores the variate in `held` (a retry after the static tier gives up overwrites it) and the
// body folds `held` after the hold.  Kind 100 exists only here: cmb_random_flip() and then an exponential in one sampler, so a
// give-up on the static tier must put back the flip cache as well as the generator.
// counters: [0] an order-dependent fold of the body's bit patterns, h = (h ^ bits) * 0x100000001b3 + 1 from 0xcbf29ce484222325;
// [1] the first and [2] the last bit pattern; [3] min and [4] max (NaN skipped) as bits; [5] draws; [6] NaNs; [7] the same fold
// over the held durations (0xcbf29ce484222325 when there were none).  objects = draws; t_end = the clock after the holds.
#pragma once
#include "../cimba_b200/csrc/cmb_kernel.cuh"
#include "../cimba_b200/csrc/cmb_static.cuh"
#include "random_sweep_table.h"

namespace random_sweep {
using namespace cimba_b200;

constexpr uint64_t FOLD_START = 0xcbf29ce484222325ull;

CMB_FN uint64_t fold_in(uint64_t h, double v)
{
    return (h ^ (uint64_t)__double_as_longlong(v)) * 0x100000001b3ull + 1ull;
}

template <class S>
struct SweepT {
    uint32_t kind, np, held_ok;
    double   p[MAXP];
    cmb_random_alias<MAXP> table;
    uint64_t i, fold, fold_held, first, last, count, nans;
    double   lo, hi, held;
    static CMB_FN constexpr uint32_t static_kind(uint32_t) { return 0u; }
    static constexpr bool static_interrupts = true;        // the tier's form with cmb_random_flip's cache (StaticSim<..., PRE = true>)

    CMB_FN double draw(S &sim)
    {
        const unsigned cnt = (unsigned)p[0];
        switch (kind) {
        case 9:  return cmb_random_triangular(p[0], p[1], p[2]);
        case 10: return cmb_random_lognormal(p[0], p[1]);
        case 11: return cmb_random_logistic(p[0], p[1]);
        case 12: return cmb_random_cauchy(p[0], p[1]);
        case 13: return cmb_random_hypoexponential(cnt, p + 1);
        case 14: return cmb_random_hyperexponential(cnt, p + 1, p + 1 + cnt);
        case 15: return cmb_random_gamma(p[0], p[1]);
        case 16: return cmb_random_beta(p[0], p[1], p[2], p[3]);
        case 17: return cmb_random_PERT(p[0], p[1], p[2]);
        case 18: return cmb_random_weibull(p[0], p[1]);
        case 19: return cmb_random_pareto(p[0], p[1]);
        case 20: return cmb_random_chisquared(p[0]);
        case 21: return cmb_random_F_dist(p[0], p[1]);
        case 22: return cmb_random_t_dist(p[0], p[1], p[2]);
        case 23: return cmb_random_rayleigh(p[0]);
        case 24: return (double)cmb_random_flip();
        case 25: return (double)cmb_random_geometric(p[0]);
        case 26: return (double)cmb_random_binomial(cnt, p[1]);
        case 27: return (double)cmb_random_negative_binomial(cnt, p[1]);
        case 28: return (double)cmb_random_poisson(p[0]);
        case 29: return (double)cmb_random_loaded_dice(cnt, p + 1);
        case 30: return (double)cmb_random_alias_sample(table);
        case 31: return cmb_random_std_gamma(p[0]);
        case 32: return cmb_random_PERT_mod(p[0], p[1], p[2], p[3]);
        case 33: return (double)cmb_random_pascal(cnt, p[1]);
        case 100: {
            const double f = (double)cmb_random_flip();
            return f + cmb_random_std_exponential();
        }
        default: return 0.0;
        }
    }

    CMB_FN void record(double v)
    {
        const uint64_t b = (uint64_t)__double_as_longlong(v);
        fold = fold_in(fold, v);
        if (count == 0u) first = b;
        last = b;
        count++;
        if (v != v) {
            nans++;
        }
        else {
            if (v < lo) lo = v;
            if (v > hi) hi = v;
        }
    }

    CMB_FN void body(S &sim, uint32_t me, int64_t sig)
    {
        SweepT &m = *this;
        CMB_PROCESS_BEGIN
        for (i = 0u; i < NDRAW; i++) {
            record(draw(sim));
        }
        if (held_ok) {
            for (i = 0u; i < NDRAW; i++) {
                CMB_PROCESS_HOLD_SAMPLED(0u);
                fold_held = fold_in(fold_held, held);
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN double sample(S &sim, uint32_t)
    {
        held = draw(sim);
        return held;
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        const Case &c = CASES[in.trial < NCASES ? in.trial : 0u];
        kind = c.kind;
        np = c.np;
        held_ok = c.held;
        for (uint32_t k = 0u; k < MAXP; k++) p[k] = c.p[k];
        if (kind == 30u) cmb_random_alias_create(table, (unsigned)p[0], p + 1);
        fold = fold_held = FOLD_START;
        first = last = count = nans = 0u;
        lo = __longlong_as_double(0x7ff0000000000000ll);
        hi = -lo;
        held = 0.0;
        cmb_process_start(cmb_process_create(0u, 0, 0u));
    }
    CMB_FN void process(S &sim, uint32_t me, uint32_t, int64_t sig) { body(sim, me, sig); }
    CMB_FN void event(S &, uint32_t, uint32_t, int64_t) {}
    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }
    CMB_FN void finish(S &, cmb::TrialOut &out)
    {
        out.objects = count;
        out.sum_wait = 0.0;
        out.max_queue = 0u;
        out.counters[0] = fold;
        out.counters[1] = first;
        out.counters[2] = last;
        out.counters[3] = (uint64_t)__double_as_longlong(lo);
        out.counters[4] = (uint64_t)__double_as_longlong(hi);
        out.counters[5] = count;
        out.counters[6] = nans;
        out.counters[7] = fold_held;
    }
};
}  // namespace random_sweep
