// distributions.cuh - the rest of cmb_random on the device.
//
// Reference: include/cmb_random.h:189-940 and src/cmb_random.c:299-313, 465-766.  Every
// function is a thin layer over sfc64 and the two ziggurats (rng.cuh), in the reference's
// draw order, so a stream seeded like the reference's yields the same variates:
//   * bit-exact by construction (sqrt and division are IEEE-exact on both sides):
//     triangular, cauchy, hypo/hyperexponential, rayleigh, flip, binomial, poisson,
//     loaded_dice, alias_sample;
//   * bit-exact in practice - log() only feeds the accept/reject comparison of the
//     Marsaglia-Tsang squeeze, so a last-place difference between CUDA's and glibc's log
//     matters only if the two sides of that comparison agree to ~1e-16:
//     std_gamma, gamma (shape >= 1), beta, PERT, chisquared (k >= 2), F, t;
//   * bit-exact because the only libm call is exp(), restated from glibc (glibc_exp.cuh): lognormal
//     (the ziggurat wedge tests in rng.cuh use the same routine);
//   * within the accuracy of CUDA's log / pow (<= 2 ulp) of the reference's glibc result,
//     because the transcendental IS the variate: logistic, weibull, pareto, gamma with
//     shape < 1 (and what builds on it); geometric / negative_binomial apply ceil() to such a
//     value and can differ by one on a measure-zero set.  glibc's log and pow tables were
//     chosen by search and cannot be recomputed from first principles, so they stay CUDA's.
// Compiled with -fmad=false: the expressions keep the reference's operation order.
#pragma once

#include <cmath>
#include <cstdint>

#include "rng.cuh"

namespace cimba_b200 {

// Out-of-line draws for the general-path kernels.  rng.cuh's members inline their ziggurat slow
// paths (exp(), alias tables, rejection loops: 400-600 instructions) into every call site, which is
// right for the small hot kernels and wrong for code that draws in dozens of places: the harbor
// kernel was 40 % inlined generator code and stalled on the instruction cache.
__device__ __noinline__ double gp_std_normal(Sfc64 &r, const ZigHot &hot)
{
    return r.std_normal(hot);
}

__device__ __noinline__ double gp_exponential(Sfc64 &r, const ZigHot &hot, double mean)
{
    return r.exponential(hot, mean);
}

__device__ __noinline__ double gp_uniform01(Sfc64 &r)
{
    return r.uniform01();
}

// ------------------------------------------------------------------------------------------------ one formulation
// Each distribution is written ONCE, below, as a template over a "sim": anything with a generator `rng` (Sfc64), its ziggurat
// tables `hot`, and the two ziggurat draws draw_exponential(s, mean) / draw_std_normal(s) found for it by argument-dependent
// lookup.  Three sims exist:
//   * GpDraws (here): a generator and its tables, as the general-path kernels and cimba_b200_rng_draws_ex hold them.  Its draws
//     are the out-of-line gp_* above, and the rnd_* functions at the end of this file are this formulation on it;
//   * cmb::Sim (cmb_device.cuh): the same out-of-line draws;
//   * cmb::StaticSim (cmb_static.cuh), which says `static constexpr bool inline_draws = true;`: inline draws that take no
//     address of the generator (a call would put the whole control block in local memory), and that GIVE UP in a sampler the
//     dispatcher is trying with the ziggurats' rectangles only (hot_only -> hot_failed).  Every loop below that draws from a
//     ziggurat leaves as soon as draw_gave_up(s) says so: the value is thrown away, the generator rewound, and the sampler
//     repeated later with the slow paths allowed.
// On the two out-of-line sims the Marsaglia-Tsang loop is one __noinline__ function (gp_std_gamma) and cmb_random() is
// gp_uniform01; on the static tier everything inlines.
template <class S, class = void>
struct InlineDraws {
    static constexpr bool value = false;
};
template <class S>
struct InlineDraws<S, decltype((void)S::inline_draws)> {
    static constexpr bool value = S::inline_draws;
};

template <class S>
__device__ __forceinline__ double draw_uniform01(S &s)
{
    if constexpr (InlineDraws<S>::value) return s.rng.uniform01();
    else return gp_uniform01(s.rng);
}

template <class S>
__device__ __forceinline__ bool draw_gave_up(const S &s)
{
    if constexpr (InlineDraws<S>::value) return s.hot_failed;
    else return false;
}

struct GpDraws {
    Sfc64         &rng;
    const ZigHot  *hot;
};

__device__ __forceinline__ double draw_exponential(GpDraws &s, double mean) { return gp_exponential(s.rng, *s.hot, mean); }
__device__ __forceinline__ double draw_std_normal(GpDraws &s) { return gp_std_normal(s.rng, *s.hot); }

// include/cmb_random.h:319-329: the exponential of mean 1 (1.0 * x is x)
template <class S>
__device__ __forceinline__ double random_std_exponential(S &s)
{
    return draw_exponential(s, 1.0);
}

// src/cmb_random.c:500-520
template <class S>
__device__ __forceinline__ double random_triangular(S &s, double min, double mode, double max)
{
    const double u = draw_uniform01(s);
    if (u < (mode - min) / (max - min)) {
        return min + sqrt(u * (max - min) * (mode - min));
    }
    return max - sqrt((1.0 - u) * (max - min) * (max - mode));
}

// include/cmb_random.h:249-257
template <class S>
__device__ __forceinline__ double random_lognormal(S &s, double m, double sd)
{
    return glibc_exp((m + sd * draw_std_normal(s)));       // the variate IS an exp: glibc's bits (glibc_exp.cuh)
}

// :267-273
template <class S>
__device__ __forceinline__ double random_logistic(S &s, double m, double sc)
{
    const double x = draw_uniform01(s);
    return m + sc * log(x / (1.0 - x));
}

// :290-299
template <class S>
__device__ __forceinline__ double random_cauchy(S &s, double mode, double scale)
{
    const double x = draw_std_normal(s);
    double y;
    while ((y = draw_std_normal(s)) == 0.0) {
        if (draw_gave_up(s)) break;
    }
    return mode + scale * x / y;
}

// :394-408
template <class S>
__device__ __forceinline__ double random_hypoexponential(S &s, unsigned n, const double *ma)
{
    double x = 0.0;
    for (unsigned i = 0u; i < n; i++) {
        x += draw_exponential(s, ma[i]);
    }
    return x;
}

// src/cmb_random.c:644-662, with one rule of this port: the result is ALWAYS < n (n >= 1; n = 0 reads nothing and gives 0, and
// model code flags the trial, cmb_device.cuh).  The reference accepts probabilities
// that sum to 1 within 1e-3 (sums_to_one) and asserts the bound in debug builds only, so a draw above a sum just under 1 returns
// n there - past the end of the array, which cmb_random_hyperexponential then reads.  Here such a draw lands on the LAST FACE
// WITH A POSITIVE PROBABILITY (face n - 1 if none has one).  Wherever the reference's result is a face, this is the same face.
template <class S>
__device__ __forceinline__ unsigned random_loaded_dice(S &s, unsigned n, const double *pa)
{
    const double x = draw_uniform01(s);
    double q = 0.0;
    unsigned last = n > 0u ? n - 1u : 0u;
    for (unsigned ui = 0u; ui < n; ui++) {
        q += pa[ui];
        if (x < q) {
            return ui;
        }
        if (pa[ui] > 0.0) {
            last = ui;
        }
    }
    return last;
}

// :299-313
template <class S>
__device__ __forceinline__ double random_hyperexponential(S &s, unsigned n, const double *ma, const double *pa)
{
    const unsigned ui = random_loaded_dice(s, n, pa);
    return n > 0u ? draw_exponential(s, ma[ui]) : 0.0;
}

// A CPU build of this text may define CMB_OBSERVE_SQUEEZE(lhs, rhs, d, log_w) to see each of the Marsaglia-Tsang loop's log
// comparisons (tests/random_sweep_host.cpp measures how close they come to a tie); elsewhere it is nothing.
#ifndef CMB_OBSERVE_SQUEEZE
#define CMB_OBSERVE_SQUEEZE(lhs, rhs, d, log_w) ((void)0)
#endif

// Marsaglia & Tsang, src/cmb_random.c:465-497
template <class S>
__device__ __forceinline__ double std_gamma_loop(S &s, double shape)
{
    const double d = shape - 1.0 / 3.0;
    const double c = 1.0 / sqrt(9.0 * d);
    double x, v;
    for (;;) {
        do {
            x = draw_std_normal(s);
            if (draw_gave_up(s)) return d;
            v = 1.0 + c * x;
        } while (v <= 0.0);
        const double w = v * v * v;
        const double u = draw_uniform01(s);
        if (u < 1.0 - 0.331 * (x * x) * (x * x)) {
            return d * w;
        }
        const double lhs = log(u);
        const double log_w = log(w);
        const double rhs = (0.5 * x * x) + (d * (1.0 - w + log_w));
        CMB_OBSERVE_SQUEEZE(lhs, rhs, d, log_w);
        if (lhs < rhs) {
            return d * w;
        }
    }
}

__device__ __noinline__ double gp_std_gamma(Sfc64 &r, const ZigHot &hot, double shape)
{
    GpDraws s{r, &hot};
    return std_gamma_loop(s, shape);
}

template <class S>
__device__ __forceinline__ double random_std_gamma(S &s, double shape)
{
    if constexpr (InlineDraws<S>::value) return std_gamma_loop(s, shape);
    else return gp_std_gamma(s.rng, *s.hot, shape);
}

// include/cmb_random.h:451-463.  For shape < 1 the reference writes
// cmb_random_std_gamma(shape + 1) * pow(cmb_random(), 1 / shape): C leaves the evaluation order of the two operands
// unspecified; gcc 13 (-O2/-O3, x86-64) - the build the oracle and the golden vectors come from - draws std_gamma
// first, and so does this.  A different compiler could legitimately produce the other stream.
template <class S>
__device__ __forceinline__ double random_gamma(S &s, double shape, double scale)
{
    if (shape >= 1.0) {
        return scale * random_std_gamma(s, shape);
    }
    const double g = random_std_gamma(s, shape + 1.0);
    const double u = draw_uniform01(s);
    return scale * (g * pow(u, 1.0 / shape));
}

// :476-487
template <class S>
__device__ __forceinline__ double random_std_beta(S &s, double a, double b)
{
    const double x = random_std_gamma(s, a);
    const double y = random_std_gamma(s, b);
    return x / (x + y);
}

// :500-512
template <class S>
__device__ __forceinline__ double random_beta(S &s, double a, double b, double min, double max)
{
    return min + (max - min) * random_std_beta(s, a, b);
}

// src/cmb_random.c:523-538; cmb_random_PERT (include/cmb_random.h:541-553) is lambda = 4
template <class S>
__device__ __forceinline__ double random_PERT_mod(S &s, double min, double mode, double max, double lambda)
{
    const double rng = max - min;
    const double a = 1.0 + lambda * (mode - min) / rng;
    const double b = 1.0 + lambda * (max - mode) / rng;
    return min + rng * random_std_beta(s, a, b);
}

// :571-582
template <class S>
__device__ __forceinline__ double random_weibull(S &s, double shape, double scale)
{
    const double u = draw_exponential(s, 1.0);
    return scale * pow(u, 1.0 / shape);
}

// :595-605
template <class S>
__device__ __forceinline__ double random_pareto(S &s, double shape, double mode)
{
    return mode / pow(draw_uniform01(s), 1.0 / shape);
}

// :618-626
template <class S>
__device__ __forceinline__ double random_chisquared(S &s, double k)
{
    return random_gamma(s, k / 2.0, 2.0);
}

// :639-653
template <class S>
__device__ __forceinline__ double random_F_dist(S &s, double a, double b)
{
    const double x = random_chisquared(s, a) / a;
    double y;
    while ((y = random_chisquared(s, b) / b) == 0.0) {
        if (draw_gave_up(s)) break;
    }
    return x / y;
}

// :668-679
template <class S>
__device__ __forceinline__ double random_std_t_dist(S &s, double v)
{
    const double x = draw_std_normal(s);
    double y;
    while ((y = random_chisquared(s, v)) == 0.0) {
        if (draw_gave_up(s)) break;
    }
    return x / sqrt(y / v);
}

// :693-702
template <class S>
__device__ __forceinline__ double random_t_dist(S &s, double m, double sc, double v)
{
    return m + sc * random_std_t_dist(s, v);
}

// :714-725
template <class S>
__device__ __forceinline__ double random_rayleigh(S &s, double sc)
{
    const double x = (0.0 + sc * draw_std_normal(s));
    const double y = (0.0 + sc * draw_std_normal(s));
    return sqrt(x * x + y * y);
}

// :558-573.  The reference returns (unsigned)ceil(...), and for p below about 1e-9 the quotient passes 2^32 (nearly always at
// p = 1e-12; p > 0 is all the reference asks).  That conversion is undefined in C (C11 6.3.1.4); the reference's build, gcc on
// x86-64, wraps it modulo 2^32 where the device's cvt.rzi.u32.f64 would saturate at 4294967295: x86_cvttsd2si (rng.cuh) states
// the wrap.
template <class S>
__device__ __forceinline__ unsigned random_geometric(S &s, double p)
{
    const double denom = -log(1.0 - p);
    return (unsigned)(uint64_t)x86_cvttsd2si(ceil(draw_exponential(s, 1.0) / denom));
}

// :576-588
template <class S>
__device__ __forceinline__ unsigned random_binomial(S &s, unsigned n, double p)
{
    unsigned k = 0u;
    for (unsigned i = 0u; i < n; i++) {
        k += s.rng.bernoulli(p);
    }
    return k;
}

// :594-606; cmb_random_pascal (include/cmb_random.h:812-815) is the same function
template <class S>
__device__ __forceinline__ unsigned random_negative_binomial(S &s, unsigned m, double p)
{
    unsigned f = 0u;
    for (unsigned i = 0u; i < m; i++) {
        f += random_geometric(s, p) - 1u;
        if (draw_gave_up(s)) break;
    }
    return f;
}

// :612-632
template <class S>
__device__ __forceinline__ unsigned random_poisson(S &s, double rate)
{
    const double m = 1.0 / rate;
    double t = 0.0;
    unsigned ctr = 0u;
    for (;;) {
        t += draw_exponential(s, m);
        if (draw_gave_up(s)) break;
        if (t <= 1.0) {
            ctr++;
        }
        else {
            break;
        }
    }
    return ctr;
}

// cmb_random_alias_sample, include/cmb_random.h:922-933, on tables from cmb_random_alias_create (AliasTable below) or
// cimba_b200_alias_create
template <class S>
__device__ __forceinline__ unsigned random_alias_sample(S &s, unsigned n, const uint64_t *uprob, const uint32_t *alias)
{
    const unsigned idx = (unsigned)floor((double)n * draw_uniform01(s));
    const bool c = s.rng.next() >= uprob[idx];
    return c ? alias[idx] : idx;
}

// cmb_random_alias_create, src/cmb_random.c:688-752 (Vose), built in place: the tables of a `struct cmb_random_alias` of at most
// N entries, as a member of a model.  Same arithmetic as the host's cimba_b200_alias_create, so the same bits.  Probabilities are
// the caller's (summing to 1 as the reference requires); create() returns false, and leaves an empty table that samples 0, when n
// is 0 or above N - model code then flags the trial (cmb_random_alias_create, cmb_device.cuh).
__host__ __device__ inline uint64_t alias_secure(double p)             // src/cmb_random.c:672-686; the host's too (capi.cu)
{
    if (p <= 0.0) return 0u;
    if (p >= 1.0) return UINT64_MAX;
    return (uint64_t)(p * 18446744073709551616.0);                      // (double)UINT64_MAX is 2^64
}

template <unsigned N>
struct AliasTable {
    uint32_t n;
    uint64_t uprob[N];
    uint32_t alias[N];

    __device__ __forceinline__ bool create(unsigned count, const double *pa)
    {
        n = (count >= 1u && count <= N) ? count : 0u;
        if (n == 0u) {
            uprob[0] = 0u;
            alias[0] = 0u;
            return false;
        }
        double work[N];
        uint32_t small_[N], large_[N];
        double psum = 0.0;
        for (uint32_t i = 0u; i < n; i++) {
            psum += pa[i];
            uprob[i] = 0u;
            alias[i] = 0u;
        }
        uint32_t ns = 0u, nl = 0u;
        for (uint32_t i = 0u; i < n; i++) {
            work[i] = pa[i] * (double)n / psum;
            if (work[i] < 1.0) small_[ns++] = i;
            else large_[nl++] = i;
        }
        while (ns > 0u && nl > 0u) {
            const uint32_t l = small_[--ns];
            const uint32_t g = large_[--nl];
            uprob[l] = alias_secure(work[l]);
            alias[l] = g;
            work[g] = (work[g] + work[l]) - 1.0;
            if (work[g] < 1.0) small_[ns++] = g;
            else large_[nl++] = g;
        }
        while (nl > 0u) uprob[large_[--nl]] = UINT64_MAX;
        while (ns > 0u) uprob[small_[--ns]] = UINT64_MAX;
        return true;
    }
};

// ------------------------------------------------------------------------------------------------ the general path's names
// The formulation above on a bare generator: cimba_b200_rng_draws_ex and the general-path kernels.
__device__ inline double rnd_triangular(Sfc64 &r, double min, double mode, double max)
{
    GpDraws s{r, nullptr};
    return random_triangular(s, min, mode, max);
}

__device__ inline double rnd_lognormal(Sfc64 &r, const ZigHot &hot, double m, double sd)
{
    GpDraws s{r, &hot};
    return random_lognormal(s, m, sd);
}

__device__ inline double rnd_logistic(Sfc64 &r, double m, double sc)
{
    GpDraws s{r, nullptr};
    return random_logistic(s, m, sc);
}

__device__ inline double rnd_cauchy(Sfc64 &r, const ZigHot &hot, double mode, double scale)
{
    GpDraws s{r, &hot};
    return random_cauchy(s, mode, scale);
}

__device__ inline double rnd_hypoexponential(Sfc64 &r, const ZigHot &hot, unsigned n, const double *ma)
{
    GpDraws s{r, &hot};
    return random_hypoexponential(s, n, ma);
}

__device__ inline unsigned rnd_loaded_dice(Sfc64 &r, unsigned n, const double *pa)
{
    GpDraws s{r, nullptr};
    return random_loaded_dice(s, n, pa);
}

__device__ inline double rnd_hyperexponential(Sfc64 &r, const ZigHot &hot, unsigned n, const double *ma, const double *pa)
{
    GpDraws s{r, &hot};
    return random_hyperexponential(s, n, ma, pa);
}

__device__ inline double rnd_std_gamma(Sfc64 &r, const ZigHot &hot, double shape)
{
    return gp_std_gamma(r, hot, shape);
}

__device__ inline double rnd_gamma(Sfc64 &r, const ZigHot &hot, double shape, double scale)
{
    GpDraws s{r, &hot};
    return random_gamma(s, shape, scale);
}

__device__ inline double rnd_std_beta(Sfc64 &r, const ZigHot &hot, double a, double b)
{
    GpDraws s{r, &hot};
    return random_std_beta(s, a, b);
}

__device__ inline double rnd_beta(Sfc64 &r, const ZigHot &hot, double a, double b, double min, double max)
{
    GpDraws s{r, &hot};
    return random_beta(s, a, b, min, max);
}

__device__ inline double rnd_PERT_mod(Sfc64 &r, const ZigHot &hot, double min, double mode, double max, double lambda)
{
    GpDraws s{r, &hot};
    return random_PERT_mod(s, min, mode, max, lambda);
}

__device__ inline double rnd_weibull(Sfc64 &r, const ZigHot &hot, double shape, double scale)
{
    GpDraws s{r, &hot};
    return random_weibull(s, shape, scale);
}

__device__ inline double rnd_pareto(Sfc64 &r, double shape, double mode)
{
    GpDraws s{r, nullptr};
    return random_pareto(s, shape, mode);
}

__device__ inline double rnd_chisquared(Sfc64 &r, const ZigHot &hot, double k)
{
    GpDraws s{r, &hot};
    return random_chisquared(s, k);
}

__device__ inline double rnd_F_dist(Sfc64 &r, const ZigHot &hot, double a, double b)
{
    GpDraws s{r, &hot};
    return random_F_dist(s, a, b);
}

__device__ inline double rnd_std_t_dist(Sfc64 &r, const ZigHot &hot, double v)
{
    GpDraws s{r, &hot};
    return random_std_t_dist(s, v);
}

__device__ inline double rnd_t_dist(Sfc64 &r, const ZigHot &hot, double m, double sc, double v)
{
    GpDraws s{r, &hot};
    return random_t_dist(s, m, sc, v);
}

__device__ inline double rnd_rayleigh(Sfc64 &r, const ZigHot &hot, double sc)
{
    GpDraws s{r, &hot};
    return random_rayleigh(s, sc);
}

// cmb_random_flip, src/cmb_random.c:541-552: 64 coin flips per sfc64 word, most significant
// bit first.  The reference keeps the cache in thread-local statics; here it is part of
// the trial's generator state.
struct FlipCache {
    uint64_t bits;
    uint32_t pos;
};

__device__ inline int rnd_flip(Sfc64 &r, FlipCache &f)
{
    if (f.pos == 0u) {
        f.bits = r.next();
        f.pos = 64u;
    }
    return (int)((f.bits >> --f.pos) & 1u);
}

__device__ inline unsigned rnd_geometric(Sfc64 &r, const ZigHot &hot, double p)
{
    GpDraws s{r, &hot};
    return random_geometric(s, p);
}

__device__ inline unsigned rnd_binomial(Sfc64 &r, unsigned n, double p)
{
    GpDraws s{r, nullptr};
    return random_binomial(s, n, p);
}

__device__ inline unsigned rnd_negative_binomial(Sfc64 &r, const ZigHot &hot, unsigned m, double p)
{
    GpDraws s{r, &hot};
    return random_negative_binomial(s, m, p);
}

__device__ inline unsigned rnd_poisson(Sfc64 &r, const ZigHot &hot, double rate)
{
    GpDraws s{r, &hot};
    return random_poisson(s, rate);
}

__device__ inline unsigned rnd_alias_sample(Sfc64 &r, unsigned n, const uint64_t *uprob, const uint32_t *alias)
{
    GpDraws s{r, nullptr};
    return random_alias_sample(s, n, uprob, alias);
}

}  // namespace cimba_b200
