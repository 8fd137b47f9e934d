// tests/random_sweep_host.cpp - TEST INFRASTRUCTURE: the cmb_random formulation (cimba_b200/csrc/distributions.cuh) and the sweep model
// (tests/random_sweep_model.cuh) compiled for the CPU, as a small C library for tests/test_random_sweep.py and
// tests/golden/make_random_sweep_golden.py:
//   * sweep_draws: n variates of one kind 9..33 (the numbering of cimba_b200_rng_draws_ex) through the general path's
//     formulation, as rng_draws_ex_kernel draws them, with the generator calls the stream made (sfc64's counter word counts
//     them) and the smallest margin, over every log comparison of the Marsaglia-Tsang loop in the stream, between its two
//     sides: |lhs - rhs| in units of the last places of the libm results that enter it (ulp(lhs) + |d| ulp(log w) + ulp(rhs)).
//     A platform whose log differs from glibc's by a few ulp takes the same branch wherever that margin is large;
//   * gamma_parts: the two factors std_gamma(shape + 1) and u of gamma's shape < 1 branch, drawn in its order;
//   * sweep_model_run: the sweep model's trials on the general engine (cmb::Sim) or on the static tier (cmb::StaticSim<1, 0>
//     through static_run_trial_host, the tier's own dispatcher: sampled holds tried with the rectangles only, and on giving up
//     the generator rewound and the sampler repeated).  random_sweep_table.h comes from the include path.
// The CUDA vocabulary is mapped to C++ as in tests/cmb_engine_host.cpp.  Not a product path: built by the tests.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC -I <table dir> random_sweep_host.cpp -o librandom_sweep_host.so
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <vector>

static double g_margin = std::numeric_limits<double>::infinity();
static uint64_t g_compares = 0u;

static double ulp_of(double x)
{
    const double a = std::fabs(x);
    return std::nextafter(a, std::numeric_limits<double>::infinity()) - a;
}

static void observe_squeeze(double lhs, double rhs, double d, double log_w)
{
    g_compares++;
    if (std::isnan(lhs) || std::isnan(rhs)) return;             // the comparison is false whatever the last places are
    const double scale = ulp_of(lhs) + std::fabs(d) * ulp_of(log_w) + ulp_of(rhs);
    const double m = std::fabs(lhs - rhs) / scale;
    if (m < g_margin) g_margin = m;
}
#define CMB_OBSERVE_SQUEEZE(lhs, rhs, d, log_w) observe_squeeze((lhs), (rhs), (d), (log_w))

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

#include "random_sweep_model.cuh"

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

constexpr unsigned PMAX = 64u;

// one variate of `kind`, as rng_draws_ex_kernel's switch draws it, on any sim of the formulation
template <class S>
double draw_kind(S &s, int kind, const double *p, const AliasTable<PMAX> &table, FlipCache &flips)
{
    const unsigned cnt = (unsigned)p[0];
    switch (kind) {
    case 9:  return random_triangular(s, p[0], p[1], p[2]);
    case 10: return random_lognormal(s, p[0], p[1]);
    case 11: return random_logistic(s, p[0], p[1]);
    case 12: return random_cauchy(s, p[0], p[1]);
    case 13: return random_hypoexponential(s, cnt, p + 1);
    case 14: return random_hyperexponential(s, cnt, p + 1, p + 1 + cnt);
    case 15: return random_gamma(s, p[0], p[1]);
    case 16: return random_beta(s, p[0], p[1], p[2], p[3]);
    case 17: return random_PERT_mod(s, p[0], p[1], p[2], 4.0);
    case 18: return random_weibull(s, p[0], p[1]);
    case 19: return random_pareto(s, p[0], p[1]);
    case 20: return random_chisquared(s, p[0]);
    case 21: return random_F_dist(s, p[0], p[1]);
    case 22: return random_t_dist(s, p[0], p[1], p[2]);
    case 23: return random_rayleigh(s, p[0]);
    case 24: return (double)rnd_flip(s.rng, flips);
    case 25: return (double)random_geometric(s, p[0]);
    case 26: return (double)random_binomial(s, cnt, p[1]);
    case 27: return (double)random_negative_binomial(s, cnt, p[1]);
    case 28: return (double)random_poisson(s, p[0]);
    case 29: return (double)random_loaded_dice(s, cnt, p + 1);
    case 30: return (double)random_alias_sample(s, table.n, table.uprob, table.alias);
    case 31: return random_std_gamma(s, p[0]);
    case 32: return random_PERT_mod(s, p[0], p[1], p[2], p[3]);
    case 33: return (double)random_negative_binomial(s, cnt, p[1]);
    default: return 0.0;
    }
}
}  // namespace

// n variates of `kind` (params p[0..np)) from a generator seeded `seed` through GpDraws (cimba_b200_rng_draws_ex's
// formulation).  *calls = generator calls of the stream, *margin = its smallest squeeze margin (infinity when it made no log
// comparison), *compares = how many it made.  -1 for an unknown kind or too many parameters.
extern "C" int sweep_draws(uint64_t seed, int kind, const double *pp, uint32_t np, uint64_t n, double *general, uint64_t *calls,
                           double *margin, uint64_t *compares)
{
    if (kind < 9 || kind > 33 || np > PMAX) return -1;
    double p[PMAX] = {0};
    for (uint32_t i = 0; i < np; i++) p[i] = pp[i];
    AliasTable<PMAX> table;
    table.n = 0u;
    if (kind == 30 && !table.create((unsigned)p[0], p + 1)) return -1;
    const ZigHot &hot = host_hot();

    Sfc64 r;
    r.seed(seed);
    const uint64_t d0 = r.d;
    GpDraws g{r, &hot};
    FlipCache flips{0u, 0u};
    g_margin = std::numeric_limits<double>::infinity();
    g_compares = 0u;
    for (uint64_t i = 0; i < n; i++) general[i] = draw_kind(g, kind, p, table, flips);
    *calls = r.d - d0;
    *margin = g_margin;
    *compares = g_compares;
    return 0;
}

struct HostResult {
    uint64_t events, objects;
    double   t_end, sum_wait;
    uint64_t counter[8];
    uint32_t status, pad;
};

// trials [0, count) of the sweep model, seeds cmb_random_fmix64(master_seed, i): engine 0 = the general engine, 1 = the static
// tier.  -1 for another engine.
extern "C" int sweep_model_run(int engine, uint64_t master_seed, uint64_t count, HostResult *out)
{
    if (engine < 0 || engine > 1) return -1;
    const ZigHot &hot = host_hot();
    static std::vector<unsigned char> mem(1u << 20);
    for (uint64_t i = 0; i < count; i++) {
        cmb::TrialIn in{};
        in.num_objects = 0u;
        in.servers = 1;
        in.trial = i;
        const uint64_t seed = fmix64(master_seed, i);
        cmb::TrialOut o;
        HostResult &r = out[i];
        if (engine == 0) {
            unsigned long long cursor = 0;
            cmb::Arena arena{mem.data(), &cursor, mem.size()};
            static cmb::Sim sim;
            static random_sweep::SweepT<cmb::Sim> m;
            sim.init(seed, &hot, arena);
            cmb::run_one_trial<random_sweep::SweepT<cmb::Sim>, false>(sim, m, in, o, 0u, nullptr, nullptr);
            r.events = sim.pops;
            r.t_end = sim.now;
            r.status = sim.status;
        }
        else {
            using S = cmb::StaticFormOf<random_sweep::SweepT, 1, 0, 1>;
            static S sim;
            static random_sweep::SweepT<S> m;
            static double win[cmb::STATIC_WINDOW];
            sim.init(seed, &hot, win, 1u, nullptr, 0u);
            cmb::static_run_trial_host(sim, m, in, o, 0u, nullptr, nullptr);
            r.events = sim.pops;
            r.t_end = sim.now;
            r.status = sim.status;
        }
        r.objects = o.objects;
        r.sum_wait = o.sum_wait;
        std::memcpy(r.counter, o.counters, sizeof r.counter);
        r.pad = 0u;
    }
    return 0;
}

// gamma's shape < 1 branch, factor by factor: g[i] = std_gamma(shape + 1), u[i] = the uniform drawn after it
extern "C" int gamma_parts(uint64_t seed, double shape, uint64_t n, double *g, double *u)
{
    const ZigHot &hot = host_hot();
    Sfc64 r;
    r.seed(seed);
    for (uint64_t i = 0; i < n; i++) {
        g[i] = rnd_std_gamma(r, hot, shape + 1.0);
        u[i] = r.uniform01();
    }
    return 0;
}
