// tests/model_random_host.cpp - TEST INFRASTRUCTURE: the cmb_random distributions, alias tables and summaries of model code,
// compiled for the CPU from the same source text as the device's, as a small C library for tests/test_model_random.py:
//   * every distribution drawn through the general path's formulation (GpDraws, what rnd_* and cmb::Sim use) and through the
//     static tier's (cmb::StaticSim), the latter as the dispatcher draws a sampler: rectangles only first, and when that gives
//     up the generator rewound and the draw repeated with the slow paths;
//   * cmb_random_loaded_dice / _hyperexponential on a generator that returns the largest uniform there is;
//   * cmb_random_alias_create's tables, and cmb_datasummary / cmb_wtdsummary through the model-code names;
//   * examples/clinic_model.cuh on the general engine and on cmb::StaticSim<4, 2>, as tests/static_coverage_host.cpp runs its
//     models.
// The CUDA vocabulary is mapped to C++ as in tests/cmb_engine_host.cpp.  Not a product path: built by the test.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC model_random_host.cpp -o libmodel_random_host.so
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define CMB_HOST_BUILD 1
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __fma_rn(double a, double b, double c) { return std::fma(a, b, c); }
static inline double __ull2double_rn(unsigned long long v) { return (double)v; }
static inline double __ll2double_rn(long long v) { return (double)v; }
static inline long long __double_as_longlong(double d) { long long i; std::memcpy(&i, &d, 8); return i; }
static inline double __longlong_as_double(long long i) { double d; std::memcpy(&d, &i, 8); return d; }
static inline double __hiloint2double(int hi, int lo)
{
    const unsigned long long b = ((unsigned long long)(unsigned)hi << 32) | (unsigned)lo;
    double d; std::memcpy(&d, &b, 8); return d;
}
static inline int __double2hiint(double d) { return (int)((unsigned long long)__double_as_longlong(d) >> 32); }
static inline int __double2loint(double d) { return (int)(unsigned)__double_as_longlong(d); }
struct HostDim3 { unsigned x, y, z; };
static HostDim3 threadIdx = {0, 0, 0}, blockDim = {1, 1, 1};
template <class T> static inline T max(T a, T b) { return a < b ? b : a; }
static inline unsigned long long __cvta_generic_to_shared(const void *p) { return (unsigned long long)(uintptr_t)p; }

#include "../examples/clinic_model.cuh"

using namespace cimba_b200;

namespace {
ZigHot &host_hot()
{
    static ZigHot hot;
    static bool ready = false;
    if (!ready) {
        for (int i = 0; i < 256; i++) {
            hot.exp_x[i] = zig::zig_exp_x[i];
            hot.nor_x[i] = zig::zig_nor_x[i];
        }
        ready = true;
    }
    return hot;
}

const double HYPO_M[3] = {0.5, 1.0, 2.0};
const double HYPER_M[3] = {0.3, 1.0, 4.0};
const double HYPER_P[3] = {0.6, 0.3, 0.1};
const double DICE_P[4] = {0.1, 0.2, 0.3, 0.4};

// kind -> one variate; the same list in tests/test_model_random.py
template <class S>
double draw_kind(S &s, int kind, const AliasTable<5> &table)
{
    switch (kind) {
    case 0:  return random_std_exponential(s);
    case 1:  return random_triangular(s, 1.0, 2.0, 4.0);
    case 2:  return random_lognormal(s, 0.1, 0.5);
    case 3:  return random_logistic(s, 0.0, 1.0);
    case 4:  return random_cauchy(s, 0.0, 1.0);
    case 5:  return random_hypoexponential(s, 3u, HYPO_M);
    case 6:  return random_hyperexponential(s, 3u, HYPER_M, HYPER_P);
    case 7:  return random_std_gamma(s, 2.5);
    case 8:  return random_gamma(s, 0.5, 2.0);
    case 9:  return random_gamma(s, 3.5, 0.5);
    case 10: return random_std_beta(s, 2.0, 3.0);
    case 11: return random_beta(s, 0.5, 0.7, 1.0, 3.0);
    case 12: return random_PERT_mod(s, 1.0, 2.0, 5.0, 4.0);
    case 13: return random_weibull(s, 1.5, 2.0);
    case 14: return random_pareto(s, 3.0, 1.0);
    case 15: return random_chisquared(s, 3.0);
    case 16: return random_F_dist(s, 5.0, 10.0);
    case 17: return random_std_t_dist(s, 4.0);
    case 18: return random_t_dist(s, 1.0, 2.0, 5.0);
    case 19: return random_rayleigh(s, 1.5);
    case 20: return (double)random_geometric(s, 0.3);
    case 21: return (double)random_binomial(s, 10u, 0.3);
    case 22: return (double)random_negative_binomial(s, 3u, 0.4);
    case 23: return (double)random_poisson(s, 4.5);
    case 24: return (double)random_loaded_dice(s, 4u, DICE_P);
    case 25: return (double)random_alias_sample(s, table.n, table.uprob, table.alias);
    case 26: return random_chisquared(s, 1.0);
    default: return 0.0;
    }
}

// a generator whose every uniform is the largest below 1, and whose exponentials are their means
struct TopUniform {
    double uniform01() { return 1.0 - 0x1p-53; }
};
struct TopSim {
    static constexpr bool inline_draws = true;
    TopUniform rng;
    bool hot_failed = false;
};
double draw_exponential(TopSim &, double mean) { return mean; }
double draw_std_normal(TopSim &) { return 0.0; }
}  // namespace

extern "C" int host_random_kinds() { return 27; }

// n variates of `kind` from a generator seeded `seed`: general[] through GpDraws, stat[] through cmb::StaticSim in the
// dispatcher's manner; *rewinds = how many static draws gave up on the rectangles and were repeated
extern "C" int host_random_streams(int kind, uint64_t seed, uint64_t n, double *general, double *stat, uint64_t *rewinds)
{
    if (kind < 0 || kind >= host_random_kinds()) return -1;
    const ZigHot &hot = host_hot();
    AliasTable<5> table;
    const double ap[5] = {0.05, 0.4, 0.15, 0.3, 0.1};
    table.create(5u, ap);
    Sfc64 r;
    r.seed(seed);
    GpDraws g{r, &hot};
    for (uint64_t i = 0; i < n; i++) general[i] = draw_kind(g, kind, table);

    using Static = cmb::StaticSim<1, 0>;
    static Static sim;
    double win[cmb::STATIC_WINDOW];
    sim.init(seed, &hot, win, 1u, nullptr, 0u);
    *rewinds = 0u;
    for (uint64_t i = 0; i < n; i++) {
        const Sfc64 saved = sim.rng;
        sim.hot_only = true;
        sim.hot_failed = false;
        double v = draw_kind(sim, kind, table);
        sim.hot_only = false;
        if (sim.hot_failed) {
            sim.hot_failed = false;
            sim.rng = saved;
            v = draw_kind(sim, kind, table);
            *rewinds += 1u;
        }
        stat[i] = v;
    }
    return 0;
}

// cmb_random_loaded_dice(n, pa) and cmb_random_hyperexponential(n, ma, pa) when the uniform lies above the probabilities' sum;
// ma[n] is the caller's sentinel, which must not be read
extern "C" void host_dice_bound(unsigned n, const double *pa, const double *ma, unsigned *face, double *hyper)
{
    TopSim s;
    *face = random_loaded_dice(s, n, pa);
    *hyper = random_hyperexponential(s, n, ma, pa);
}

// cmb_random_alias_create(a, n, pa) into a table of capacity 64; -1 when it refuses n
extern "C" int host_alias_create(unsigned n, const double *pa, uint64_t *uprob, uint32_t *alias)
{
    AliasTable<64> a;
    if (!a.create(n, pa) || a.n != n) return -1;         // n = 0 or above the capacity: refused
    for (unsigned i = 0; i < n; i++) {
        uprob[i] = a.uprob[i];
        alias[i] = a.alias[i];
    }
    return 0;
}

// the model-code summary calls over x[0..n) (weights w[0..n) for the weighted kind, halves merged at k); out = {count, min, max,
// m1, m2, m3, m4, wsum} of the merged summary then {mean, variance, stddev, skewness, kurtosis}; row = cmb_summary_to_counters
extern "C" void host_summaries(int weighted, uint64_t n, uint64_t k, const double *x, const double *w, double *out, uint64_t *row)
{
    cmb::TrialOut o{};
    if (!weighted) {
        cmb_datasummary a, b, c;
        cmb_datasummary_initialize(&a);
        cmb_datasummary_initialize(&b);
        for (uint64_t i = 0; i < n; i++) (void)cmb_datasummary_add(i < k ? &a : &b, x[i]);
        (void)cmb_datasummary_merge(&c, &a, &b);
        const double v[13] = {(double)cmb_datasummary_count(&c), cmb_datasummary_min(&c), cmb_datasummary_max(&c), c.m1, c.m2, c.m3,
                              c.m4, 0.0, cmb_datasummary_mean(&c), cmb_datasummary_variance(&c), cmb_datasummary_stddev(&c),
                              cmb_datasummary_skewness(&c), cmb_datasummary_kurtosis(&c)};
        std::memcpy(out, v, sizeof v);
        cmb_summary_to_counters(o, &c);
    }
    else {
        cmb_wtdsummary a, b, c;
        cmb_wtdsummary_initialize(&a);
        cmb_wtdsummary_initialize(&b);
        for (uint64_t i = 0; i < n; i++) (void)cmb_wtdsummary_add(i < k ? &a : &b, x[i], w[i]);
        (void)cmb_wtdsummary_merge(&c, &a, &b);
        const double v[13] = {(double)cmb_wtdsummary_count(&c), cmb_wtdsummary_min(&c), cmb_wtdsummary_max(&c), c.m1, c.m2, c.m3,
                              c.m4, c.wsum, cmb_wtdsummary_mean(&c), cmb_wtdsummary_variance(&c), cmb_wtdsummary_stddev(&c),
                              cmb_wtdsummary_skewness(&c), cmb_wtdsummary_kurtosis(&c)};
        std::memcpy(out, v, sizeof v);
        cmb_summary_to_counters(o, &c);
    }
    std::memcpy(row, o.counters, sizeof o.counters);
}

// ---- the clinic on both engines
struct HostResult {
    uint64_t events, objects;
    double   t_end, sum_wait;
    uint64_t max_fel, max_queue;
    uint64_t counter[8];
    uint32_t status, pad;
};

template <class S>
static void copy_out(const S &sim, const cmb::TrialOut &out, HostResult &r)
{
    r.events = sim.pops;
    r.objects = out.objects;
    r.t_end = sim.now;
    r.sum_wait = out.sum_wait;
    r.max_fel = 0u;
    r.max_queue = out.max_queue;
    std::memcpy(r.counter, out.counters, sizeof(r.counter));
    r.status = sim.status;
    r.pad = 0u;
}

// engine 0 = the general engine (arena_bytes of growth memory), 1 = the static tier as examples/clinic_static_user_model.cu
// builds it.  trace_cap pops of each trial into trace_key / trace_time [count][trace_cap].  Returns 0, -1 for another engine.
extern "C" int host_clinic_run_trials(int engine, uint64_t master_seed, uint64_t first, uint64_t count, uint64_t num_objects,
                                      double arr_mean, double srv_mean, double report, uint64_t arena_bytes, uint64_t trace_cap,
                                      uint64_t *trace_key, double *trace_time, HostResult *out)
{
    if (engine < 0 || engine > 1) return -1;
    const ZigHot &hot = host_hot();
    std::vector<unsigned char> mem((engine == 0 ? arena_bytes : 0u) + 256);
    for (uint64_t i = 0; i < count; i++) {
        cmb::TrialIn in{};
        in.arr_mean = arr_mean;
        in.srv_mean = srv_mean;
        in.num_objects = num_objects;
        in.servers = 1;
        in.trial = first + i;
        in.num_params = 1u;
        in.params[0] = report;
        const uint64_t seed = fmix64(master_seed, first + i);
        uint64_t *tk = trace_cap ? trace_key + i * trace_cap : nullptr;
        double *tt = trace_cap ? trace_time + i * trace_cap : nullptr;
        cmb::TrialOut o;
        if (engine == 0) {
            unsigned long long cursor = 0;
            cmb::Arena arena{mem.data(), &cursor, arena_bytes};
            static cmb::Sim sim;
            static clinic_example::ClinicT<cmb::Sim> m;
            sim.init(seed, &hot, arena);
            if (trace_cap) cmb::run_one_trial<clinic_example::ClinicT<cmb::Sim>, true>(sim, m, in, o, trace_cap, tk, tt);
            else           cmb::run_one_trial<clinic_example::ClinicT<cmb::Sim>, false>(sim, m, in, o, 0u, nullptr, nullptr);
            copy_out(sim, o, out[i]);
        }
        else {
            using S = cmb::StaticSim<4, 2>;
            static S sim;
            static clinic_example::ClinicT<S> m;
            static double win[2 * cmb::STATIC_WINDOW];
            static double spill[2 * 4096];
            sim.init(seed, &hot, win, 1u, spill, 4096u);
            cmb::static_run_trial_host(sim, m, in, o, trace_cap, tk, tt);
            copy_out(sim, o, out[i]);
        }
    }
    return 0;
}
